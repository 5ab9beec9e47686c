"""DPRDistillTask - drop-in for ``dpr_scale.task.dpr_distill_task.DPRDistillTask``: one query encoder trained with
``MSELoss(reduction="sum")`` toward target vectors (typically a DrBoost ensemble's embeddings of the question and of
one of its positive passages), so that query time runs one encoder instead of K.

Same constructor keywords, Lightning hook names and metric names as the reference.  What changed:

  * the encoder is ``dpr_scale_b200.models.hf_model.HFEncoder`` (libdprb.so kernels);
  * the loss and its gradient are one pass of ``dprb_sqerr_fwd`` (``_SqErr``); evaluation scores the query
    representations against the targets with the fused scoring kernel and ranks with the DPR task's device-side rule.
"""
import torch
from torch.optim.lr_scheduler import LambdaLR

from .. import ops
from ..utils.config import instantiate
from ..utils.lightning_shim import LightningModule
from .dpr_task import DenseRetrieverTask


class _SqErr(torch.autograd.Function):
    """loss = sum (x - t)^2 with dx = 2 (x - t) written by the same kernel pass; targets get no gradient."""

    @staticmethod
    def forward(ctx, x, t):
        loss_sum, ctx.dx = ops.sqerr(x.detach(), t.detach(), want_dx=True)
        return loss_sum[0]

    @staticmethod
    def backward(ctx, g):
        dx = ctx.dx * g
        ctx.dx = None
        return dx, None


def encoder_out_dim(encoder):
    """Width of an HFEncoder's output: the projection dim, else the hidden size."""
    proj = encoder.project
    return proj[0].out_features if isinstance(proj, torch.nn.Sequential) else encoder.config["hidden_size"]


class DPRDistillTask(LightningModule):
    def __init__(
        self,
        transform,
        model,
        datamodule,
        optim,
        warmup_steps: int = 0,
        fp16_grads: bool = False,
        pretrained_checkpoint_path: str = "",
        k=1,
    ):
        super().__init__()
        self.save_hyperparameters()
        self.transform_conf = transform.text_transform if hasattr(transform, "text_transform") else transform
        self.model_conf = model
        self.optim_conf = optim
        self.k = k
        self.warmup_steps = warmup_steps
        self.fp16_grads = fp16_grads
        self.pretrained_checkpoint_path = pretrained_checkpoint_path
        self.setup_done = False

    def setup(self, stage: str):
        if stage == "test" and self.setup_done:
            return
        self.call_configure_sharded_model_hook = False
        self.query_encoder = instantiate(self.model_conf)
        if self.pretrained_checkpoint_path:
            ckpt = torch.load(self.pretrained_checkpoint_path, map_location="cpu", weights_only=False)
            self.load_state_dict(ckpt["state_dict"])
            print(f"Loaded state dict from {self.pretrained_checkpoint_path}")
        self.setup_done = True

    def on_load_checkpoint(self, checkpoint) -> None:
        self.setup("fit")

    def on_pretrain_routine_start(self):
        # as in DenseRetrieverTask: `fp16_grads` selects the trainer's bf16-compressed gradient all-reduce
        if self.trainer is not None and hasattr(self.trainer, "set_grad_compression"):
            self.trainer.set_grad_compression(bool(self.fp16_grads))

    # ------------------------------------------------------------------ encoder
    def _encode_sequence(self, token_ids, encoder_model):
        return encoder_model(token_ids)

    def encode_queries(self, query_ids):
        return self._encode_sequence(query_ids, self.query_encoder)

    def forward(self, query_ids):
        return self.encode_queries(query_ids)

    def _targets(self, batch):
        """fp32 targets on the encoder's device; a width that differs from the encoder's output is refused before any
        GPU work."""
        targets = batch["target_vectors"]
        width = encoder_out_dim(self.query_encoder)
        if targets.dim() != 2 or targets.shape[1] != width:
            raise ValueError(f"distillation targets are {tuple(targets.shape)} but the query encoder outputs {width} "
                             "values per question: the target width must equal the projection dim (or the hidden size "
                             "without a projection)")
        return targets.to(self.query_encoder.master.device, torch.float32)

    # ------------------------------------------------------------------ optimizer / schedule
    def configure_optimizers(self):
        self.optimizer = instantiate(self.optim_conf, self.parameters())
        if hasattr(self.optimizer, "attach_encoders"):
            self.optimizer.attach_encoders([self.query_encoder])
        if self.trainer.max_steps and self.trainer.max_steps > 0:
            training_steps = self.trainer.max_steps
        else:
            training_steps = len(self.trainer.datamodule.train_dataloader()) * self.trainer.max_epochs
        print(f"Configured LR scheduler for total {training_steps} training steps, "
              f"with {self.warmup_steps} warmup steps.")
        warm = self.warmup_steps

        def lr_lambda(step):
            if step < warm:
                return float(step) / float(max(1, warm))
            return max(0.0, float(training_steps - step) / float(max(1, training_steps - warm)))

        sched = {"scheduler": LambdaLR(self.optimizer, lr_lambda), "name": "learning_rate", "interval": "step",
                 "frequency": 1}
        return [self.optimizer], [sched]

    # ------------------------------------------------------------------ training / evaluation
    def training_step(self, batch, batch_idx):
        targets = self._targets(batch)
        query_repr = self(batch["query_ids"])
        loss = _SqErr.apply(query_repr, targets.contiguous())
        self.log("train_loss", loss, prog_bar=True)
        return loss

    def _eval_step(self, batch, batch_idx):
        targets = self._targets(batch).contiguous()
        query_repr = self(batch["query_ids"]).contiguous()
        labels = torch.arange(targets.shape[0], device=targets.device)
        _, _, scores, _ = ops.score_fwd(query_repr, targets, None, labels, 1.0, True)
        loss_sum, _ = ops.sqerr(query_repr, targets, want_dx=False)
        return (DenseRetrieverTask.compute_rank_metrics(self, scores, labels), query_repr, targets, loss_sum[0])

    def _eval_epoch_end(self, outputs, log_prefix="valid"):
        total_loss, total_mrr, total_avg_rank, total_score, total_ctx_count, total_count = 0, 0, 0, 0, 0, 0
        for metrics, query_repr, targets, loss in outputs:
            rank, mrr, score = metrics
            total_avg_rank += rank
            total_mrr += mrr
            total_count += query_repr.shape[0]
            total_ctx_count += targets.shape[0]
            total_score += score
            total_loss += loss
        total_loss = total_loss / len(outputs)
        total_ctx_count = total_ctx_count / len(outputs)
        metrics = {
            log_prefix + "_loss": total_loss,
            log_prefix + f"_accuracy@{self.k}": total_score / total_count,
            log_prefix + "_avg_rank": total_avg_rank / total_count,
            log_prefix + "_mrr": total_mrr / total_count,
            log_prefix + "_ctx_count": total_ctx_count,
        }
        self.log_dict(metrics, on_epoch=True, sync_dist=True)
        return metrics

    def validation_step(self, batch, batch_idx):
        return self._eval_step(batch, batch_idx)

    def validation_epoch_end(self, valid_outputs):
        return self._eval_epoch_end(valid_outputs) if valid_outputs else None

    def test_step(self, batch, batch_idx):
        return self._eval_step(batch, batch_idx)

    def test_epoch_end(self, test_outputs):
        return self._eval_epoch_end(test_outputs, "test") if test_outputs else None
