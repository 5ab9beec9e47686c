"""CrossEncoderTrainTask: fine-tunes the cross-encoder that ``task=cross_encoder_rerank`` runs.  The reference ships the
batches for this (``DPRCrossAttentionTransform``, selected by ``use_cross_attention``) but its CrossEncoderTask has no
training step; this task adds one.

Each batch holds B groups of G (question, passage) pairs whose pair 0 is relevant (``datamodule=cross_encoder_train``).
The loss is the mean over groups of the softmax cross-entropy of the group's relevance logits
(``CrossEncoder.group_ce``: the fused ``dprb_seqcls_group_ce`` head kernel, the library's GEMMs and HFEncoder's
backward).  The optimizer and the warmup + linear-decay schedule are DenseRetrieverTask's, with the fused optimizers
attached to the body's parameter arena; under DDP the trainer all-reduces the arena by layer buckets during backward and
the head's parameters after it, as for the DPR task.  Groups never cross ranks: every row of a batch is one group.

Validation and test log ``<split>_loss`` (mean over groups), ``<split>_avg_rank`` and ``<split>_mrr`` of the relevant
pair among its group (DenseRetrieverTask's tie rule: an equal score ranks it behind the pairs before it) and
``<split>_accuracy`` (its share in the top ``k``), summed over every rank.  A checkpoint holds CrossEncoderTask's
``state_dict`` keys, so it loads strictly into ``task=cross_encoder_rerank`` through ``task.pretrained_checkpoint_path``.
"""
import torch
import torch.distributed as dist

from .cross_encoder_task import CrossEncoderTask
from .dpr_task import DenseRetrieverTask


class CrossEncoderTrainTask(CrossEncoderTask):
    def __init__(self, transform, model, datamodule, optim, k=1, shared_model: bool = True, in_batch_eval: bool = True,
                 warmup_steps: int = 0, fp16_grads: bool = False, pretrained_checkpoint_path: str = ""):
        super().__init__(transform, model, datamodule, optim, k, shared_model, in_batch_eval, warmup_steps, fp16_grads,
                         pretrained_checkpoint_path)
        self.optim_conf = optim
        self.warmup_steps = warmup_steps or 0

    # the arena-backed encoder, under the names the trainer's gradient buckets and the fused optimizers look up
    @property
    def query_encoder(self):
        return self.cross_encoder._body

    @property
    def context_encoder(self):
        return self.cross_encoder._body

    configure_optimizers = DenseRetrieverTask.configure_optimizers
    on_pretrain_routine_start = DenseRetrieverTask.on_pretrain_routine_start
    compute_rank_metrics = DenseRetrieverTask.compute_rank_metrics

    def training_step(self, batch, batch_idx):
        loss, _ = self.cross_encoder.group_ce(batch["text_ids"], batch["labels"], batch["group_size"])
        self.log("train_loss", loss, prog_bar=True)
        return loss

    def _eval_step(self, batch, batch_idx):
        G = int(batch["group_size"])
        loss, logits = self.cross_encoder.group_ce(batch["text_ids"], batch["labels"], G)
        labels = torch.as_tensor(batch["labels"]).to(logits.device, torch.int64)
        rank, mrr, hits = self.compute_rank_metrics(logits.view(-1, G), labels)
        return rank, mrr, hits, labels.numel(), float(loss) * labels.numel()

    def _eval_epoch_end(self, outputs, prefix):
        totals = torch.tensor([sum(o[i] for o in outputs) for i in range(5)], dtype=torch.float64)
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            dev = torch.device("cuda", torch.cuda.current_device()) if dist.get_backend() == "nccl" else None
            totals = totals.to(dev)
            dist.all_reduce(totals)
            totals = totals.cpu()
        rank, mrr, hits, n, loss = totals.tolist()
        metrics = {prefix + "_loss": loss / n, prefix + "_avg_rank": rank / n, prefix + "_mrr": mrr / n,
                   prefix + "_accuracy": hits / n}
        self.log_dict(metrics, on_epoch=True)
        return metrics

    def validation_step(self, batch, batch_idx):
        return self._eval_step(batch, batch_idx)

    def validation_epoch_end(self, outputs):
        return self._eval_epoch_end(outputs, "valid") if outputs else None

    def test_step(self, batch, batch_idx):
        return self._eval_step(batch, batch_idx)

    def test_epoch_end(self, outputs):
        return self._eval_epoch_end(outputs, "test") if outputs else None
