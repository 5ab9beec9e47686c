"""Retrieval from a COIL / CITADEL expert index: drop-in for the reference's ``CITADELRetrievalTask``
(dpr_scale/task/citadel_retrieval_task.py, config conf/task/multivec_retrieval.yaml), whose search lives in an inverted
vector index module that its tree does not contain.

``ExpertIndex`` reads what GenerateMultiVecEmbeddingsTask writes (``expert_{rank}/{expert}.pkl`` and ``cls_{rank}.pkl``)
for a passage table of N rows and searches it on the device with ``dprb_expert_search``:

  score(q, d) = cls_q . cls_d                                               (only with add_cls)
              + sum over q's entries (x, u) of max(0, max over d's index entries (x, v) of u . v)    (max over {} = 0)

Query entries are the reference's (its ``_eval_step``): the unmasked tokens 1.. (COIL), or every expert slot with a
positive weight (CITADEL), payload ``weight * rep``.  Payloads and CLS vectors are fp16 on the device, products are
fp32-accumulated, terms are summed as int64 fixed point at 2^-32, so two runs give identical results and a query's
results do not depend on the other queries of its batch.  Ranking: descending score, ties towards the lower passage
row; the returned ids are the corpus ids of the index files.

Device memory: about E * (2 * P16 + 4) + N * (2 * Pc16 + 8) bytes for the index (E entries, P16 / Pc16 = P / Pc rounded
up to 16, and the int64 corpus id of every row) plus the query-block accumulator of at most 2 GiB, which
``ops.expert_search`` keeps cached per device for the life of the process.
"""
import concurrent.futures
import glob
import json
import os
import pickle
import time

import numpy as np
import torch
import torch.distributed as dist

from .. import ops
from ..datamodule.cross_encoder import IDCSVDataset
from ..models.citadel_models.coil_model import COILEncoder
from .citadel_eval_task import MultiVecRetrieverTask


def _pad16(n):
    return (n + 15) // 16 * 16


def _load(path):
    with open(path, "rb") as f:
        return pickle.load(f)


def passage_ids(table):
    """int64 [N]: the ``id`` column of a passage table (an IDCSVDataset), in row order (ValueError: a non-integer
    id)."""
    out = np.empty(table.count - 1, dtype=np.int64)
    for i in range(1, table.count):
        pid = table.process_line(table._row(i))["id"]
        try:
            out[i - 1] = int(pid)
        except ValueError:
            raise ValueError(f"passage id {pid!r} is not an integer (expert indexes use integer corpus ids)") from None
    return out


class ExpertIndex:
    """A COIL / CITADEL expert index on one device, searched with ``dprb_expert_search``.

    Build it from files with ``ExpertIndex.load`` or from arrays with the constructor.  ``search`` takes the
    query entries grouped by expert (``ops.expert_group`` with ``per_sequence=False``) and returns the k best passages
    of every query."""

    READERS = 16

    def __init__(self, expert, row, payload, ids, cls=None, V=None, device="cuda"):
        """expert / row: host int arrays [E] (row = passage row in [0, N)), payload [E, P] (float tensor or array, any
        device), ids int64 [N] (corpus id of every row), cls [N, Pc] or None, V: the expert vocabulary."""
        t0 = time.perf_counter()
        expert = np.asarray(expert, dtype=np.int64)
        row = np.asarray(row, dtype=np.int64)
        ids = np.asarray(ids, dtype=np.int64)
        payload = torch.as_tensor(payload)
        N, E = ids.size, expert.size
        if payload.dim() != 2 or payload.shape[0] != E:
            raise ValueError(f"expert index payload must be [E={E}, P] vectors (got {tuple(payload.shape)}); an "
                             "add_context_id index holds token ids, not vectors, and cannot be searched")
        P = int(payload.shape[1])
        V = int(expert.max()) + 1 if V is None and E else int(V or 1)
        Pc = None if cls is None else int(cls.shape[1])
        ops.expert_search_check(P, Pc, V, E, max(N, 1), 1)
        if E and (expert.min() < 0 or expert.max() >= V):
            raise ValueError(f"expert ids must lie in [0, {V})")
        if E and (row.min() < 0 or row.max() >= N):
            raise ValueError(f"passage rows must lie in [0, {N})")
        if cls is not None and cls.shape[0] != N:
            raise ValueError(f"the index has {cls.shape[0]} CLS rows for a table of {N} passages")
        order = None
        key = expert * N + row
        if E > 1 and bool(np.any(key[1:] < key[:-1])):
            order = np.argsort(key, kind="stable")     # by expert, then row; the generation order is kept otherwise
            expert, row = expert[order], row[order]
        self.device = torch.device(device)
        self.N, self.E, self.P, self.Pc, self.V = N, E, P, Pc, V
        self.tile_bounds_host, self.tile_ptr = ops.expert_search_tiles(expert, row, V)
        pay = payload if order is None else payload[torch.from_numpy(order).to(payload.device)]
        self.payload, self.max_norm = self._to_fp16(pay, "index payload")
        self.row = torch.from_numpy(row.astype(np.int32)).to(self.device)
        self.tile_bounds = torch.from_numpy(self.tile_bounds_host).to(self.device)
        self.ids = torch.from_numpy(ids).to(self.device)
        self.cls, self.cls_max_norm = (None, 0.0) if cls is None else self._to_fp16(torch.as_tensor(cls), "CLS vector")
        self.load_seconds = time.perf_counter() - t0

    CHUNK = 1 << 18                                   # rows converted at a time: bounded temporaries

    def _to_fp16(self, x, what):
        """fp16 [n, width16] on the device (zero-padded columns) and the largest row norm; ValueError when a value does
        not fit fp16.  Host input is converted and checked on the host in chunks and copied to the device once."""
        n, w = x.shape
        out = torch.zeros(max(n, 1), _pad16(w), dtype=torch.float16, device=x.device)
        norm = 0.0
        for a in range(0, n, self.CHUNK):
            c = x[a:a + self.CHUNK].float()
            if not bool(torch.isfinite(c).all()) or float(c.abs().max()) > ops.FP16_MAX:
                raise ValueError(f"a {what} does not fit fp16 (|value| > {ops.FP16_MAX:g} or not finite)")
            h = c.half()
            out[a:a + self.CHUNK, :w] = h
            norm = max(norm, float(h.float().norm(dim=1).max()))
        return out.to(self.device), norm

    @classmethod
    def load(cls, ctx_embeddings_dir, ids, add_cls=False, P=None, Pc=None, device="cuda", workers=None):
        """Read every ``expert_*/`` shard and the ``cls_*.pkl`` files in rank order (a bounded thread pool) for the
        passage table whose corpus ids are ``ids`` (int [N], row order).  ValueError: an id not in the table, a CLS
        row count other than N, add_cls without CLS files, a payload width other than the encoder's P (or Pc), or an
        add_context_id index."""
        ids = np.asarray(ids, dtype=np.int64)
        shards = sorted(glob.glob(os.path.join(ctx_embeddings_dir, "expert_*")))
        files = [(x, os.path.join(d, f"{x}.pkl")) for d in shards
                 for x in sorted(int(n[:-4]) for n in os.listdir(d) if n.endswith(".pkl"))]
        with concurrent.futures.ThreadPoolExecutor(max_workers=workers or cls.READERS) as pool:
            parts = list(pool.map(lambda xf: _load(xf[1]), files))
        experts, cids, pays = [], [], []
        for (x, path), (cid, _w, pay) in zip(files, parts):
            if pay.dim() != 2:
                raise ValueError(f"{path} holds token ids, not vectors: an add_context_id index cannot be searched")
            if P is not None and pay.shape[1] != P:
                raise ValueError(f"{path} holds {pay.shape[1]}-wide payloads but the encoder's are {P}-wide")
            experts.append(np.full(len(cid), x, dtype=np.int64))
            cids.append(cid.numpy().astype(np.int64))
            pays.append(pay)
        expert = np.concatenate(experts) if experts else np.zeros(0, np.int64)
        cid = np.concatenate(cids) if cids else np.zeros(0, np.int64)
        payload = torch.cat(pays) if pays else torch.zeros(0, P or 8)
        order = np.argsort(expert, kind="stable")           # by expert; shards (ranks) keep their order
        expert, cid, payload = expert[order], cid[order], payload[torch.from_numpy(order)]
        sorter = np.argsort(ids, kind="stable")
        pos = np.searchsorted(ids, cid, sorter=sorter) if ids.size else np.zeros(cid.size, np.int64)
        pos = np.minimum(pos, max(ids.size - 1, 0))
        rows = sorter[pos] if ids.size else pos
        bad = ~(ids[rows] == cid) if ids.size else np.ones(cid.size, bool)
        if bad.any():
            raise ValueError(f"corpus id {int(cid[np.flatnonzero(bad)[0]])} of the index is not in the passage table")
        cls_vec = None
        cls_files = sorted(glob.glob(os.path.join(ctx_embeddings_dir, "cls_*.pkl")))
        if add_cls:
            if not cls_files:
                raise ValueError(f"add_cls is set but {ctx_embeddings_dir} has no cls_*.pkl files")
            cls_vec = torch.cat([_load(p).float() for p in cls_files])
            if cls_vec.shape[0] != ids.size:
                raise ValueError(f"the index has {cls_vec.shape[0]} CLS rows for a table of {ids.size} passages")
            if Pc is not None and cls_vec.shape[1] != Pc:
                raise ValueError(f"the index's CLS vectors are {cls_vec.shape[1]}-wide but the encoder's are {Pc}-wide")
        return cls(expert, rows, payload, ids, cls_vec, None if not expert.size else int(expert.max()) + 1, device)

    def search(self, q_expert, q_seq, q_payload, q_cls, n_queries, k):
        """k best passages of ``n_queries`` queries.  Query entries sorted by expert (ties in query order): q_expert
        int [Eq] (host or device), q_seq int [Eq] (query of each entry), q_payload float [Eq, P]; q_cls [n, Pc] or
        None (ignored without index CLS vectors).  Returns host (scores fp32 [n, k], corpus ids int64 [n, k])."""
        ops.expert_search_check(self.P, self.Pc, self.V, self.E, self.N, int(k))
        dev = self.device
        q_expert = torch.as_tensor(q_expert).cpu().numpy().astype(np.int64)
        q_seq_h = torch.as_tensor(q_seq).cpu().numpy().astype(np.int64)
        if q_payload.shape[1] != self.P:
            raise ValueError(f"query payloads are {q_payload.shape[1]}-wide but the index's are {self.P}-wide")
        qp, _ = self._to_fp16(torch.as_tensor(q_payload), "query payload")
        use_cls = self.cls is not None
        qc = None
        if use_cls:
            if q_cls is None or q_cls.shape != (n_queries, self.Pc):
                raise ValueError(f"the index has CLS vectors: give the queries' CLS vectors [{n_queries}, {self.Pc}]")
            qc, _ = self._to_fp16(torch.as_tensor(q_cls), "query CLS vector")
        # range of the int64 fixed point: each query's sum of |terms| stays below 2^30 (Cauchy-Schwarz)
        norms = qp.float().norm(dim=1)[:q_expert.size].cpu().numpy().astype(np.float64) if q_expert.size else np.zeros(0)
        reach = np.bincount(q_seq_h, weights=norms * self.max_norm, minlength=n_queries)
        if use_cls:
            reach = reach + qc.float().norm(dim=1)[:n_queries].cpu().numpy() * self.cls_max_norm
        if reach.size and float(reach.max()) >= ops.EXPERT_SEARCH_TERM_LIMIT:
            raise ValueError("query and index vectors are too large for the search's fixed-point sums (a query's sum "
                             f"of |u||v| reaches {float(reach.max()):.3g} >= 2^30)")
        Qb = min(ops.expert_search_block_queries(self.N), max(n_queries, 1))
        scores = np.empty((n_queries, k), np.float32)
        ids = np.empty((n_queries, k), np.int64)
        for q0 in range(0, n_queries, Qb):
            q1 = min(q0 + Qb, n_queries)
            sel = np.flatnonzero((q_seq_h >= q0) & (q_seq_h < q1))
            groups, item_end, items = ops.expert_search_groups(q_expert[sel], self.tile_ptr, q1 - q0 if use_cls else 0,
                                                               self.N)
            sel_d = torch.from_numpy(sel).to(dev)
            bp = qp[sel_d] if sel.size else qp[:1]
            bs = torch.from_numpy((q_seq_h[sel] - q0).astype(np.int32)).to(dev)
            s, i = ops.expert_search(self.payload, self.row, self.tile_bounds, self.P, self.cls, self.ids, bp, bs,
                                     None if qc is None else qc[q0:q1].contiguous(), q1 - q0,
                                     torch.from_numpy(groups).to(dev), torch.from_numpy(item_end).to(dev), items, k)
            scores[q0:q1] = s.cpu().numpy()
            ids[q0:q1] = i.cpu().numpy()
        return scores, ids


class CITADELRetrievalTask(MultiVecRetrieverTask):
    """Drop-in for the reference's ``CITADELRetrievalTask``: ``setup`` strictly loads ``checkpoint_path`` and then the
    whole index of ``ctx_embeddings_dir`` for the ``passages`` table; every rank searches its contiguous slice of the
    queries and writes ``output_path/retrieval_{rank:04}.trec`` (queries with topic ids) or ``.json`` (queries with
    answers) in the reference's formats.  ``index2docid_path`` maps the returned corpus ids to document ids."""

    def __init__(self, ctx_embeddings_dir, checkpoint_path, index2docid_path=None, hnsw_index=False,
                 output_path="/tmp/results.jsonl", passages="", topk=100, cuda=True, portion=1.0, quantizer=None,
                 sub_vec_dim=4, expert_parallel=True, **kwargs):
        super().__init__(**kwargs)
        self.ctx_embeddings_dir = ctx_embeddings_dir
        self.checkpoint_path = checkpoint_path
        self.index2docid_path = index2docid_path
        self.hnsw_index = hnsw_index
        self.output_path = output_path
        self.passages = passages
        self.topk = topk
        self.use_cuda = cuda                     # not self.cuda: that would hide nn.Module.cuda()
        self.quantizer = quantizer if quantizer != "None" else None
        self.sub_vec_dim = sub_vec_dim
        self.portion = portion
        self.expert_parallel = expert_parallel
        self.check_options()

    def check_options(self):
        """ValueError for the reference options whose behaviour lives in its missing index module."""
        if self.quantizer == "pq":
            raise ValueError("quantizer='pq' (product-quantised postings) is not supported: the index is searched "
                             "exactly, with fp16 payloads")
        if not self.use_cuda:
            raise ValueError("cuda=False is not supported: the expert index is searched on the GPU")
        if float(self.portion) != 1.0:
            raise ValueError(f"portion={self.portion} is not supported: the whole index is searched (portion=1.0)")
        if self.hnsw_index:
            raise ValueError("hnsw_index=True is not supported by multi-vector retrieval")

    def setup(self, stage: str):
        if self.setup_done:
            return
        super().setup(stage)
        self.check_encoder()
        print(f"Loading passages from {self.passages}")
        try:
            self.ctxs = IDCSVDataset(self.passages)
        except TypeError:                            # a row whose field count differs from the header's
            raise ValueError(f"{self.passages}: a row does not have the header's columns") from None
        self.passage_ids = passage_ids(self.ctxs)
        P, Pc = self._widths()
        print("Setting up index...")
        self.index = ExpertIndex.load(self.ctx_embeddings_dir, self.passage_ids, self.add_cls, P,
                                      Pc if self.add_cls else None, device=self._device())

    def check_encoder(self):
        if not hasattr(self.query_encoder, "expert_reps"):
            raise ValueError(f"multi-vector retrieval needs a COIL or CITADEL encoder (got "
                             f"{type(self.query_encoder).__name__}, which has no expert ids)")

    def _device(self):
        p = next(self.parameters(), None)
        return p.device if p is not None and p.is_cuda else torch.device("cuda", torch.cuda.current_device())

    def _widths(self):
        enc = self.query_encoder
        proj = enc.project if isinstance(enc, COILEncoder) else enc.tok_project
        P = proj[0].out_features if isinstance(proj, torch.nn.Sequential) else enc.config["hidden_size"]
        cproj = getattr(enc, "cls_project", None)
        Pc = cproj[0].out_features if isinstance(cproj, torch.nn.Sequential) else enc.config["hidden_size"]
        return P, Pc

    def query_entries(self, query_ids):
        """The query entries of one batch grouped by expert: (expert, seq, payload fp32 [Eq, P], cls [n, Pc] or None) on
        the device; seq is the query's position in the batch."""
        if torch.is_grad_enabled():
            raise ValueError("multi-vector retrieval runs forward only: call it under torch.no_grad()")
        self.check_encoder()
        enc = self.query_encoder
        am = torch.as_tensor(query_ids["attention_mask"])
        N, S = am.shape
        coil = isinstance(enc, COILEncoder)
        P, _ = self._widths()
        V = enc.config["vocab_size"]
        ops.expert_group_check(N, S, 1 if coil else int(self.query_topk), P, V)
        reps, ids, w, cls = enc.expert_reps(query_ids, topk=self.query_topk, add_cls=self.add_cls)
        expert, seq, _tok, _w, payload = ops.expert_group(reps, ids, w, am.to(reps.device), V, 0.0, None, False)
        return expert, seq, payload, cls

    def _eval_step(self, batch, batch_idx):
        query_ids = batch["query_ids"]
        topic_ids = batch["topic_ids"] if "topic_ids" in batch else []
        answers = batch["answers"] if "answers" in batch else []
        questions = batch["question"] if "question" in batch else []
        n = len(query_ids["input_ids"])
        expert, seq, payload, cls = self.query_entries(query_ids)
        scores, ids = self.index.search(expert, seq, payload, cls, n, int(self.topk))
        return scores.tolist(), ids.tolist(), list(topic_ids), list(questions), list(answers)

    def test_step(self, batch, batch_idx):
        with torch.no_grad():
            return self._eval_step(batch, batch_idx)

    def test_epoch_end(self, queries_reprs):
        top_scores, top_ids, topic_ids, questions, answers = [], [], [], [], []
        for s, i, t, q, a in queries_reprs:
            top_scores.extend(s)
            top_ids.extend(i)
            topic_ids.extend(t)
            questions.extend(q)
            answers.extend(a)
        path = None
        if len(topic_ids) > 0:
            lines = self.merge_trec_results(topic_ids, top_ids, top_scores)
            os.makedirs(self.output_path, exist_ok=True)
            path = os.path.join(self.output_path, f"retrieval_{self.global_rank:04}.trec")
            print(f"Writing output to {self.output_path}")
            with open(path, "w") as g:
                g.writelines(lines)
        elif len(answers) > 0:
            qa = self.merge_qa_results(questions, answers, top_ids, top_scores)
            os.makedirs(self.output_path, exist_ok=True)
            path = os.path.join(self.output_path, f"retrieval_{self.global_rank:04}.json")
            print(f"Writing output to {self.output_path}")
            with open(path, "w") as g:
                g.write(json.dumps(qa, indent=4))
                g.write("\n")
        if dist.is_available() and dist.is_initialized():
            dist.barrier()                       # rank 0 leaves only once every rank's file is written
        return path

    def merge_trec_results(self, topic_ids, top_doc_ids, scores_list):
        """``topic Q0 doc rank score dpr-scale`` lines; doc = line ``id`` of index2docid_path when it exists."""
        i2d = []
        if self.index2docid_path is not None and os.path.exists(self.index2docid_path):
            with open(self.index2docid_path) as f:
                i2d = [line.strip() for line in f.readlines()]
        assert len(top_doc_ids) == len(topic_ids) == len(scores_list)
        out = []
        for topic_id, doc_ids, scores in zip(topic_ids, top_doc_ids, scores_list):
            for rank, (doc_id, score) in enumerate(zip(doc_ids, scores)):
                doc = i2d[doc_id] if len(i2d) > 0 else doc_id
                out.append(f"{topic_id} Q0 {doc} {rank + 1} {score:.6f} dpr-scale\n")
        return out

    def merge_qa_results(self, questions, answers, top_doc_ids, scores_list):
        """One ``{"question", "answers", "ctxs": [{"id", "title", "text", "score"}]}`` dict per query."""
        assert len(top_doc_ids) == len(answers) == len(scores_list)
        out = []
        for question, answer, doc_ids, scores in zip(questions, answers, top_doc_ids, scores_list):
            ctxs = [{"id": self.ctxs[str(i)]["id"], "title": self.ctxs[str(i)]["title"],
                     "text": self.ctxs[str(i)]["text"], "score": float(s)} for i, s in zip(doc_ids, scores)]
            out.append({"question": question, "answers": answer, "ctxs": ctxs})
        return out
