"""Input pipeline of multi-vector (ColBERT) reranking with the interface of the reference's
``dpr_scale.datamodule.citadel.DenseRetrieverRerankDataModule`` (/root/reference/dpr_scale/datamodule/citadel.py:199-266).

The rows are those of cross-encoder reranking - one per line of a TREC run file, joined with its question and passage by
the readers of datamodule/cross_encoder.py - but questions and passages are tokenised SEPARATELY (each padded to the
longest of the batch): a batch is ``{"qid", "ctx_id", "query_ids", "contexts_ids"}``.  Under torchrun every rank reads
one contiguous, unpadded slice of the run file (ContiguousDistributedSamplerForTest).
"""
from ..transforms.dpr_transform import maybe_add_title
from .cross_encoder import TRECDataset
from .dpr import DenseRetrieverQueriesDataModule as _QueriesDataModule
from .dpr import _EncodeOnlyDataModule


class DenseRetrieverRerankDataModule(_EncodeOnlyDataModule):
    """Same keywords as the reference, plus ``prefetch_batches`` (0 = synchronous) and ``device_prefetch`` (stage
    batches on the GPU from the background thread)."""

    def __init__(self, transform, test_path: str, test_question_path: str, test_passage_path: str,
                 test_batch_size: int = 128, num_workers: int = 0, use_title: bool = False, sep_token: str = " [SEP] ",
                 query_trec: bool = True, prefetch_batches: int = 4, device_prefetch: bool = True, *args, **kwargs):
        super().__init__(transform)
        self.test_batch_size = test_batch_size
        self.use_title = use_title
        self.sep_token = sep_token
        self.num_workers = num_workers     # accepted; assembly runs on the BatchStream thread
        self.prefetch_batches, self.device_prefetch = prefetch_batches, device_prefetch
        self.datasets = {"test": TRECDataset(test_path, test_question_path, test_passage_path, query_trec)}

    def collate(self, batch, stage):
        question_tensors = self._transform([row["question"] for row in batch])
        ctx_tensors = self._transform([maybe_add_title(row["text"], row["title"], self.use_title, self.sep_token)
                                       for row in batch])
        return {"qid": [row["qid"] for row in batch], "ctx_id": [row["ctx_id"] for row in batch],
                "query_ids": question_tensors, "contexts_ids": ctx_tensors}


class DenseRetrieverQueriesDataModule(_QueriesDataModule):
    """Question file for multi-vector query embedding generation (the reference's
    ``dpr_scale.datamodule.citadel.DenseRetrieverQueriesDataModule``, datamodule/citadel.py:138-196): the readers and
    contiguous shards of the dense one, and the reference's collate: ``query_ids`` and ``question``, plus ``topic_ids``
    when the rows have ids (``trec_format``) and ``answers`` when they have answers."""

    def collate(self, batch, stage):
        inputs = {"query_ids": self._encode([row["question"] for row in batch]),
                  "question": [row["question"] for row in batch]}
        if "id" in batch[0]:
            inputs["topic_ids"] = [row["id"] for row in batch]
        if "answers" in batch[0]:
            inputs["answers"] = [row["answers"] for row in batch]
        return inputs
