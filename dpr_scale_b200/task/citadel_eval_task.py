"""Multi-vector eval tasks.  GenerateMultiVecEmbeddingsTask / GenerateMultiVecQueryEmbeddingsTask (COIL / CITADEL
expert-index generation) are documented below; the rest of this docstring is about the reranker.

RerankMultiVecRetrieverTask — drop-in for ``dpr_scale.task.citadel_eval_task.RerankMultiVecRetrieverTask``
(/root/reference/dpr_scale/task/citadel_eval_task.py:215-313) with ColBERT, COIL or CITADEL encoders: scores every
(query, passage) row
of a TREC run by late interaction and writes ``scores_{rank:04}.pkl`` (fp32 CPU tensor ``[n]``), ``qids_{rank:04}.pkl``
and ``ctx_ids_{rank:04}.pkl`` (lists), pickle protocol 4, in the row order of the rank's shard.
``python -m dpr_scale_b200.rerank`` merges them into a run file.

Accepts the keywords of the reference's ``MultiVecRetrieverTask`` (dpr_scale/task/citadel_task.py:8-24) on top of
DenseRetrieverTask's; ``query_pool`` ("sum" or "max"), ``add_cls`` and ``query_topk`` / ``context_topk`` (the experts
per CITADEL token) change what an eval step computes - the others belong to training.  ColBERT ignores the last
three, as in the reference.  ``setup`` builds the two encoders and strictly loads
``checkpoint_path`` (a Lightning checkpoint with a ``state_dict``).

An eval step never materialises ``expert_repr``: each distinct query of the batch is encoded once (rows are encoded
independently at the batch's padded width, so this equals encoding every row), the passages are encoded, both are
projected by the library's GEMM, and ``dprb_maxsim_fwd`` scores the pairs from the unmasked tokens and the masks.
With COIL / CITADEL encoders (those with ``expert_reps``) the encoders also give each token's expert ids and weights
(the mask for COIL, the router's top-k for CITADEL) and, with ``add_cls``, a CLS vector, and
``dprb_maxsim_expert_fwd`` scores the pairs with the expert-matching rule and the CLS term.
"""
import collections
import concurrent.futures
import os
import pathlib
import pickle

import numpy as np
import torch
import torch.distributed as dist

from .. import ops
from ..models.citadel_models.coil_model import COILEncoder
from .dpr_task import DenseRetrieverTask
from .rerank_common import distinct_queries, write_rerank_pickles


class MultiVecRetrieverTask(DenseRetrieverTask):
    """The keywords of the reference's ``MultiVecRetrieverTask`` (dpr_scale/task/citadel_task.py:8-24) on top of
    DenseRetrieverTask's, and the forward-only ``setup`` the multi-vector eval tasks share: build the two encoders and
    strictly load ``checkpoint_path`` (a Lightning checkpoint with a ``state_dict``)."""

    def __init__(self, add_cls: bool = False, query_topk: int = 1, context_topk: int = 1,
                 query_expert_load_loss_coef: float = 0, context_expert_load_loss_coef: float = 0,
                 query_router_marg_load_loss_coef: float = 0, context_router_marg_load_loss_coef: float = 0,
                 cross_batch: bool = True, in_batch: bool = True, query_pool: str = "sum", anneal_factor: float = 0.0,
                 teacher_coef: float = 0.0, tau: float = 1.0, **kwargs):
        super().__init__(**kwargs)
        self.query_pool = query_pool
        self.add_cls = add_cls
        self.query_topk, self.context_topk = query_topk, context_topk

    def setup(self, stage: str):
        if self.setup_done:
            return
        super().setup("train")
        print(f"Loading checkpoint from {self.checkpoint_path}")
        ckpt = torch.load(self.checkpoint_path, map_location="cpu", weights_only=False)
        self.load_state_dict(ckpt["state_dict"])


class RerankMultiVecRetrieverTask(MultiVecRetrieverTask):
    def __init__(self, checkpoint_path, output_dir, **kwargs):
        super().__init__(**kwargs)
        self.checkpoint_path = checkpoint_path
        self.output_dir = output_dir
        self.dedupe_queries = True      # False: encode every row's query (the same scores, bit for bit)
        os.makedirs(output_dir, exist_ok=True)

    def _scores(self, batch):
        if self.query_pool not in ops.MAXSIM_POOLS:
            raise NotImplementedError("Invalid query pooling! Available: [max, sum]")
        c_tok = batch["contexts_ids"]
        q_tok, index = distinct_queries(batch["qid"], batch["query_ids"], self.dedupe_queries)
        with torch.no_grad():
            if hasattr(self.query_encoder, "expert_reps"):                       # COIL / CITADEL
                q, q_ids, q_w, q_cls = self.query_encoder.expert_reps(q_tok, topk=self.query_topk, add_cls=self.add_cls)
                d, d_ids, d_w, d_cls = self.context_encoder.expert_reps(c_tok, topk=self.context_topk,
                                                                        add_cls=self.add_cls)
                return ops.maxsim_expert(q, d, q_ids, q_w, d_ids, d_w, index, self.query_pool, q_cls, d_cls)
            q, q_mask = self.query_encoder.token_reps(q_tok)
            d, d_mask = self.context_encoder.token_reps(c_tok)
            return ops.maxsim(q, d, q_mask, d_mask, index, self.query_pool)

    def _eval_step(self, batch, batch_idx):
        return [batch["qid"], batch["ctx_id"], self._scores(batch).cpu()]

    def test_step(self, batch, batch_idx):
        return self._eval_step(batch, batch_idx)

    def test_epoch_end(self, test_outputs):
        return write_rerank_pickles(self.output_dir, self.global_rank, test_outputs)


class GenerateMultiVecEmbeddingsTask(MultiVecRetrieverTask):
    """Drop-in for the reference's ``GenerateMultiVecEmbeddingsTask`` (dpr_scale/task/citadel_eval_task.py:16-117): a
    COIL or CITADEL context encoder turns the passages of ``batch["contexts_ids"]`` / ``batch["corpus_ids"]`` into an
    expert index.  Writes ``<ctx_embeddings_dir>/expert_{rank:04}/{expert}.pkl`` = (LongTensor corpus ids, fp32 weights
    [n], fp32 reprs [n, P] = weight * token rep, or [n] token ids with ``add_context_id``) per expert, entries in
    (batch, passage, token, expert slot) order, and with ``add_cls`` ``cls_{rank:04}.pkl`` = fp32 [passages, Pc].

    Kept entries follow the reference: token 0 never; COIL: unmasked tokens with weight > 0; CITADEL: unmasked tokens'
    experts with weight > ``weight_threshold``, or every expert of an unmasked token with ``add_context_id``.

    Each step encodes under no_grad, groups the batch's kept entries by expert with ``dprb_expert_group`` and copies
    them into pinned host blocks without waiting; the blocks (about E * (4P + 16) bytes for E entries) are merged into
    per-expert files at the end of the epoch by a bounded thread pool."""

    WRITERS = 16

    def __init__(self, ctx_embeddings_dir, checkpoint_path, add_context_id, weight_threshold=0., **kwargs):
        super().__init__(**kwargs)
        self.ctx_embeddings_dir = ctx_embeddings_dir
        self.checkpoint_path = checkpoint_path
        self.add_context_id = add_context_id
        self.weight_threshold = weight_threshold
        pathlib.Path(ctx_embeddings_dir).mkdir(parents=True, exist_ok=True)

    def _group(self, encoder, tokens, topk, threshold, context_id, per_sequence):
        """Encode and group one batch; returns (host block dict, cls fp32 [N, Pc] on the device or None)."""
        if not hasattr(encoder, "expert_reps"):
            raise ValueError(f"multi-vector index generation needs a COIL or CITADEL encoder (got "
                             f"{type(encoder).__name__}, which has no expert ids)")
        if torch.is_grad_enabled():
            raise ValueError("multi-vector index generation runs forward only: call it under torch.no_grad()")
        am = torch.as_tensor(tokens["attention_mask"])
        N, S = am.shape
        V = encoder.config["vocab_size"]
        coil = isinstance(encoder, COILEncoder)
        proj = encoder.project if coil else encoder.tok_project
        P = proj[0].out_features if isinstance(proj, torch.nn.Sequential) else encoder.config["hidden_size"]
        ops.expert_group_check(N, S, 1 if coil else int(topk), P, V, context_id)
        reps, ids, w, cls = encoder.expert_reps(tokens, topk=topk, add_cls=self.add_cls)
        dev = reps.device
        toks = torch.as_tensor(tokens["input_ids"]).to(dev) if context_id else None
        expert, seq, tok, weight, payload = ops.expert_group(None if context_id else reps, ids, w, am.to(dev), V,
                                                             threshold, toks, per_sequence)
        block = {}
        for name, t in (("expert", expert), ("seq", seq), ("weight", weight), ("payload", payload)):
            host = torch.empty(t.shape, dtype=t.dtype, pin_memory=t.is_cuda)
            host.copy_(t, non_blocking=True)
            block[name] = host
        ev = None
        if dev.type == "cuda":
            ev = torch.cuda.Event()
            ev.record()
        block["event"] = ev
        return block, None if cls is None else cls.float()

    def _eval_step(self, batch, batch_idx):
        corpus_ids = np.array([int(c) for c in batch["corpus_ids"]], dtype=np.int64)   # ValueError: not an integer
        coil = isinstance(self.context_encoder, COILEncoder)
        context_id = bool(self.add_context_id) and not coil
        threshold = 0.0 if coil else float(self.weight_threshold)
        block, cls = self._group(self.context_encoder, batch["contexts_ids"], self.context_topk, threshold,
                                 context_id, False)
        block["corpus_ids"] = corpus_ids
        return block, (None if cls is None else cls.cpu())

    def test_step(self, batch, batch_idx):
        return self._eval_step(batch, batch_idx)

    def test_epoch_end(self, contexts_reprs):
        if not self.ctx_embeddings_dir:
            self.ctx_embeddings_dir = getattr(self.trainer, "weights_save_path", ".")
        blocks = [_land(b) for b, _ in contexts_reprs]
        cls = [c for _, c in contexts_reprs if c is not None]
        if cls:
            cls_out_path = os.path.join(self.ctx_embeddings_dir, f"cls_{self.global_rank:04}.pkl")
            print(f"\nWriting tensors to {cls_out_path}")
            _save(cls_out_path, torch.cat(cls, 0).to(torch.float32))
        out_dir = os.path.join(self.ctx_embeddings_dir, f"expert_{self.global_rank:04}")
        print(f"\nWriting tensors to {out_dir}")
        os.makedirs(out_dir, exist_ok=True)
        write_expert_files(out_dir, blocks, self.WRITERS)
        if dist.is_available() and dist.is_initialized():
            dist.barrier()                           # rank 0 leaves only once every shard is on disk
        return out_dir


class GenerateMultiVecQueryEmbeddingsTask(GenerateMultiVecEmbeddingsTask):
    """Drop-in for the reference's ``GenerateMultiVecQueryEmbeddingsTask`` (dpr_scale/task/citadel_eval_task.py:120-213):
    the query encoder over ``batch["query_ids"]``, whose ``topic_ids`` are required.  Writes to ``query_emb_output_dir``
    (default: ``ctx_embeddings_dir``) ``query_id.pkl`` (the topic ids), ``query_repr.pkl`` and ``query_weight.pkl`` (one
    dict per query: expert -> list of fp32 tensors, [P] = weight * token rep, and the 0-d weights), and with ``add_cls``
    ``query_cls.pkl``.  Kept entries: unmasked tokens 1.. with weight > 0 (COIL weights are the mask)."""

    def __init__(self, hnsw_index=False, output_path="/tmp/results.jsonl", query_emb_output_dir=None, passages="",
                 **kwargs):
        super().__init__(**kwargs)
        self.hnsw_index = hnsw_index
        self.output_path = output_path
        self.query_emb_output_dir = query_emb_output_dir or self.ctx_embeddings_dir

    def _eval_step(self, batch, batch_idx):
        if "topic_ids" not in batch:
            raise ValueError("multi-vector query embedding generation needs topic ids: read the queries with "
                             "trec_format=true (id <tab> question)")
        topic_ids = list(batch["topic_ids"])
        block, cls = self._group(self.query_encoder, batch["query_ids"], self.query_topk, 0.0, False, True)
        block["queries"] = len(topic_ids)
        return block, topic_ids, (None if cls is None else cls.cpu())

    def test_epoch_end(self, queries_reprs):
        embeddings, weights, topic_ids, cls = [], [], [], []
        for block, b_topic_ids, b_cls in queries_reprs:
            e, w = query_dicts(_land(block))
            embeddings.extend(e)
            weights.extend(w)
            topic_ids.extend(b_topic_ids)
            if b_cls is not None:
                cls.append(b_cls)
        out_dir = self.query_emb_output_dir
        pathlib.Path(out_dir).mkdir(parents=True, exist_ok=True)
        files = [("query_id.pkl", topic_ids), ("query_repr.pkl", embeddings), ("query_weight.pkl", weights)]
        if cls:
            files.append(("query_cls.pkl", torch.cat(cls, 0)))
        for name, obj in files:
            path = os.path.join(out_dir, name)
            print(f"\nWriting tensors to {path}")
            _save(path, obj)
        return out_dir


def _save(path, obj):
    with open(path, "wb") as f:
        pickle.dump(obj, f, protocol=4)


def _land(block):
    """Wait for a block's device-to-host copies; numpy views of its arrays."""
    if block["event"] is not None:
        block["event"].synchronize()
    out = {k: (v.numpy() if torch.is_tensor(v) else v) for k, v in block.items() if k != "event"}
    return out


def write_expert_files(out_dir, blocks, workers):
    """``{expert}.pkl`` per expert of the blocks (each sorted by expert, entries in order): the blocks' entries of one
    expert are concatenated in block order (a stable sort of the concatenated expert ids)."""
    if not blocks:
        return
    experts = np.concatenate([b["expert"] for b in blocks])
    if experts.size == 0:
        return
    ids = np.concatenate([b["corpus_ids"][b["seq"]] for b in blocks])
    weights = np.concatenate([b["weight"] for b in blocks])
    payload = np.concatenate([b["payload"] for b in blocks])
    order = np.argsort(experts, kind="stable")
    sorted_experts = experts[order]
    starts = np.flatnonzero(np.r_[True, sorted_experts[1:] != sorted_experts[:-1]])
    ends = np.r_[starts[1:], sorted_experts.size]

    def write(lo, hi):
        rows = order[lo:hi]
        out = (torch.from_numpy(ids[rows]), torch.from_numpy(weights[rows]), torch.from_numpy(payload[rows]))
        _save(os.path.join(out_dir, f"{int(sorted_experts[lo])}.pkl"), out)

    with concurrent.futures.ThreadPoolExecutor(max_workers=workers) as pool:
        for f in [pool.submit(write, lo, hi) for lo, hi in zip(starts.tolist(), ends.tolist())]:
            f.result()


def query_dicts(block):
    """(embeddings, weights) of the reference's query loop for one block sorted by (query, expert): per query a
    defaultdict expert -> list of fp32 tensors ([P] payloads, 0-d weights)."""
    embeddings = [collections.defaultdict(list) for _ in range(block["queries"])]
    weights = [collections.defaultdict(list) for _ in range(block["queries"])]
    payload = torch.from_numpy(block["payload"])
    weight = torch.from_numpy(block["weight"])
    for j, (n, x) in enumerate(zip(block["seq"].tolist(), block["expert"].tolist())):
        embeddings[n][x].append(payload[j].clone())
        weights[n][x].append(weight[j].clone())
    return embeddings, weights
