"""Input pipeline of cross-encoder reranking with the interface of the reference's
``dpr_scale.datamodule.cross_encoder.CrossEncoderRerankDataModule`` (/root/reference/dpr_scale/datamodule/cross_encoder.py)
and its readers ``TRECDataset`` / ``QueryTRECDataset`` / ``IDCSVDataset`` (datamodule/citadel.py:17-132).

One row per line of a TREC run file (``qid Q0 ctx_id rank score run``); the question text is looked up by qid in a
``qid <tab> question`` file (or, with ``query_trec=False``, by row number in a question / answers file) and the passage by
id in an ``id / text / title`` table.  A batch is ``{"qid", "ctx_id", "text_ids"}`` where ``text_ids`` is the pair
tokenisation ``transform(questions, passages)`` - ``[CLS] question [SEP] passage [SEP]`` with token types 0 / 1 for a
BERT vocabulary.  Batches are assembled on BatchStream's background thread; under torchrun every rank reads one
contiguous, unpadded slice of the run file (ContiguousDistributedSamplerForTest, as in _EncodeOnlyDataModule).
"""
from ..transforms.dpr_transform import maybe_add_title
from .dpr import LineFile, QueryCSVDataset, _EncodeOnlyDataModule, _split_quoted


class _IdIndex:
    """id -> byte range of its line: the ``use_id=True`` mode of the reference's readers (citadel.py:17-77).  A repeated
    id keeps its LAST line, as the reference's offset dict does."""

    def _index_ids(self, first_row, key):
        self._by_id = {}
        for i in range(first_row, self.count):
            self._by_id[key(self._row(i))] = i

    def _row(self, i):
        return bytes(self.mm[self._bounds[i]:self._bounds[i + 1]])

    def __getitem__(self, rid):
        return self.process_line(self._row(self._by_id[rid]))


class QueryTRECDataset(_IdIndex, LineFile):
    """``qid <sep> question`` without a header, looked up by qid (citadel.py:79-108)."""

    def __init__(self, path, sep="\t"):
        LineFile.__init__(self, path, header=False)
        self.sep = sep
        self._index_ids(0, lambda line: self.process_line(line)["id"])

    def process_line(self, line):
        vals = _split_quoted(line, self.sep)
        return {"id": vals[0], "question": vals[1]}


class IDCSVDataset(_IdIndex, LineFile):
    """Delimited table with a header row, looked up by its ``id`` column (citadel.py:39-76).  A row whose field count
    differs from the header yields None, as in the reference."""

    def __init__(self, path, sep="\t"):
        LineFile.__init__(self, path, header=False)
        self.sep = sep
        self.columns = _split_quoted(self._row(0), sep) if self.count else []
        self._index_ids(1, lambda line: self.process_line(line)["id"])

    def process_line(self, line):
        vals = _split_quoted(line, self.sep)
        return dict(zip(self.columns, vals)) if len(self.columns) == len(vals) else None


class TRECDataset(LineFile):
    """Rows of a TREC run file joined with their question and passage (citadel.py:111-132)."""

    def __init__(self, path, question_path, passage_path, query_trec=True, sep=" "):
        super().__init__(path, header=False)
        self.sep = sep
        self.query_trec = query_trec
        self.question_dataset = QueryTRECDataset(question_path) if query_trec else QueryCSVDataset(question_path)
        self.passage_dataset = IDCSVDataset(passage_path)

    def process_line(self, line):
        vals = line.decode().rstrip("\r\n").split(self.sep)
        qid, ctx_id = vals[0], vals[2]
        if not self.query_trec:
            qid = int(qid)
        question = self.question_dataset[qid]
        passage = self.passage_dataset[ctx_id]
        return {"qid": qid, "ctx_id": ctx_id, "question": question["question"], "text": passage["text"],
                "title": passage["title"]}


class CrossEncoderRerankDataModule(_EncodeOnlyDataModule):
    """Same keywords as the reference, plus ``prefetch_batches`` (0 = synchronous) and ``device_prefetch`` (stage
    batches on the GPU from the background thread)."""

    def __init__(self, transform, test_path: str, test_question_path: str, test_passage_path: str,
                 test_batch_size: int = 128, num_workers: int = 0, use_title: bool = False, sep_token: str = " [SEP] ",
                 prefetch_batches: int = 4, device_prefetch: bool = True, *args, **kwargs):
        super().__init__(transform)
        self.test_batch_size = test_batch_size
        self.use_title = use_title
        self.sep_token = sep_token
        self.num_workers = num_workers     # accepted; assembly runs on the BatchStream thread
        self.prefetch_batches, self.device_prefetch = prefetch_batches, device_prefetch
        self.datasets = {"test": TRECDataset(test_path, test_question_path, test_passage_path)}

    def _transform(self, questions, ctxs):
        return self.text_transform(questions, ctxs)

    def collate(self, batch, stage):
        questions = [row["question"] for row in batch]
        ctxs = [maybe_add_title(row["text"], row["title"], self.use_title, self.sep_token) for row in batch]
        text_tensors = self._transform(questions, ctxs)
        return {"qid": [row["qid"] for row in batch], "ctx_id": [row["ctx_id"] for row in batch],
                "text_ids": text_tensors}
