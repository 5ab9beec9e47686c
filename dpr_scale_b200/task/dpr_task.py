"""DenseRetrieverTask — drop-in for ``dpr_scale.task.dpr_task.DenseRetrieverTask``
(/root/reference/dpr_scale/task/dpr_task.py:17-368) with the arithmetic on hand-written sm_90a kernels.

Same constructor kwargs, same Lightning hook names (``setup``, ``training_step``, ``validation_step`` /
``_epoch_end``, ``test_step`` / ``_epoch_end``, ``configure_optimizers``, ``on_load_checkpoint``,
``forward``, ``encode_queries``, ``encode_contexts``, ``sim_score``), same metric names.  What changed:

  * encoders are ``dpr_scale_b200.models.hf_model.HFEncoder`` (libdprb.so kernels);
  * ``sim_score`` + mask + temperature + CrossEntropyLoss (:98-105, :197-212) are ONE fused tensor-core pass
    (``dprb_score_tc_fwd``) and its backward emits only the rank-local dq / dc (:163-195 semantics);
  * the four per-tensor all-gathers of :174-176 are ONE packed NCCL all-gather.
"""
import os

import torch
import torch.distributed as dist
from torch.optim.lr_scheduler import LambdaLR

from .. import ops
from ..utils.config import instantiate
from ..utils.lightning_shim import DDPShardedStrategy, DDPStrategy, LightningModule


class _ScoreCE(torch.autograd.Function):
    """loss = mean_i CE(q_all @ c_all.T / T with masked columns, labels); grads only for the local slices.
    One fused tensor-core pass, no logits in HBM; backward recomputes the local tiles."""

    phase = None   # optional utils.phase_timer.PhaseTimer (bench.py's per-phase leg)

    @staticmethod
    def forward(ctx, q_local, c_local, q_all, c_all, labels, col_mask, pair_mask, inv_t, q0, c0):
        nq, nc = q_local.shape[0], c_local.shape[0]
        loss_sum, _, _, ctx.sctx = ops.score_fwd(q_all, c_all, col_mask, labels, inv_t, False, pair_mask, (nq, nc))
        ctx.meta = (inv_t, q0, nq, c0, nc)
        return loss_sum[0] / q_all.shape[0]

    @staticmethod
    def backward(ctx, g):
        inv_t, q0, nq, c0, nc = ctx.meta
        dq, dc = ops.score_bwd(ctx.sctx, 1.0, inv_t, q0, nq, c0, nc)
        ctx.sctx = None
        dq, dc = dq * g, dc * g
        if _ScoreCE.phase is not None:
            _ScoreCE.phase.mark("score_bwd")
        return dq, dc, None, None, None, None, None, None, None, None


class DenseRetrieverTask(LightningModule):
    def __init__(
        self,
        transform,
        model,
        datamodule,
        optim,
        k=1,
        shared_model: bool = True,
        in_batch_eval: bool = True,
        in_batch_negatives: bool = True,
        warmup_steps: int = 0,
        fp16_grads: bool = False,
        pretrained_checkpoint_path: str = "",
        softmax_temperature: float = 1.0,
    ):
        super().__init__()
        self.save_hyperparameters()
        self.transform_conf = transform.text_transform if hasattr(transform, "text_transform") else transform
        self.model_conf = model
        self.shared_model = shared_model
        self.optim_conf = optim
        self.k = k
        self.in_batch_eval = in_batch_eval
        self.in_batch_negatives = in_batch_negatives
        self.warmup_steps = warmup_steps
        self.fp16_grads = fp16_grads
        self.pretrained_checkpoint_path = pretrained_checkpoint_path
        self.softmax_temperature = softmax_temperature
        self.setup_done = False
        self.phase_timer = None   # utils.phase_timer.PhaseTimer while bench.py measures per-phase times

    # ------------------------------------------------------------------ model construction
    def setup(self, stage: str):
        if stage == "test" and self.setup_done:
            return
        self.call_configure_sharded_model_hook = False
        self.query_encoder = instantiate(self.model_conf)
        self.context_encoder = self.query_encoder if self.shared_model else instantiate(self.model_conf)
        if self.pretrained_checkpoint_path:
            ckpt = torch.load(self.pretrained_checkpoint_path, map_location="cpu", weights_only=False)
            self.load_state_dict(ckpt["state_dict"])
            print(f"Loaded state dict from {self.pretrained_checkpoint_path}")
        self.setup_done = True

    def on_load_checkpoint(self, checkpoint) -> None:
        self.setup("fit")

    def on_pretrain_routine_start(self):
        # The reference registers torch's fp16_compress_hook on the DDP wrapper (:90-92).  Here gradients are
        # reduced from the flat fp32 arena by the trainer; `fp16_grads` selects a bf16-compressed all-reduce.
        if self.trainer is not None and hasattr(self.trainer, "set_grad_compression"):
            self.trainer.set_grad_compression(bool(self.fp16_grads))

    # ------------------------------------------------------------------ encoders
    def _encode_sequence(self, token_ids, encoder_model):
        return encoder_model(token_ids)  # [n, d] fp32

    def encode_queries(self, query_ids):
        return self._encode_sequence(query_ids, self.query_encoder)

    def encode_contexts(self, contexts_ids):
        return self._encode_sequence(contexts_ids, self.context_encoder)

    def forward(self, query_ids, contexts_ids):
        # The two encoders are independent until the scoring kernel: the (8x smaller) query encoder is enqueued on a
        # side stream so its kernels fill the tail waves of the context encoder's persistent kernels; autograd replays
        # each backward on its forward stream, so the overlap also holds in backward.
        dev = getattr(self.query_encoder, "master", None)
        if (dev is not None and dev.is_cuda and self.query_encoder is not self.context_encoder
                and os.environ.get("DPRB_NO_STREAM_OVERLAP") is None):
            main = torch.cuda.current_stream()
            if getattr(self, "_side_stream", None) is None:
                self._side_stream = torch.cuda.Stream()
            side = self._side_stream
            side.wait_stream(main)
            with torch.cuda.stream(side):
                q = self.encode_queries(query_ids)
            c = self.encode_contexts(contexts_ids)
            main.wait_stream(side)
            q.record_stream(main)
            return q, c
        return self.encode_queries(query_ids), self.encode_contexts(contexts_ids)

    def sim_score(self, query_repr, context_repr, mask=None):
        """[Q, C] similarity with masked pairs set to -inf (reference :98-105), via the fused kernel."""
        q = query_repr.detach().float().contiguous()
        c = context_repr.detach().float().contiguous()
        labels = torch.zeros(q.shape[0], dtype=torch.int64, device=q.device)
        pm = None if mask is None else mask.to(q.device, torch.uint8).contiguous()
        _, _, logits, _ = ops.score_fwd(q, c, None, labels, 1.0, True, pm)
        return logits

    # ------------------------------------------------------------------ optimizer / schedule
    def configure_optimizers(self):
        self.optimizer = instantiate(self.optim_conf, self.parameters())
        if hasattr(self.optimizer, "attach_encoders"):
            self.optimizer.attach_encoders([self.query_encoder, self.context_encoder])
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

    # ------------------------------------------------------------------ training step
    def _is_ddp(self):
        return (self.trainer is not None and isinstance(getattr(self.trainer, "strategy", None),
                                                        (DDPStrategy, DDPShardedStrategy))
                and dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1)

    def _gather_global(self, q, c, labels, mask):
        """One packed all-gather of (q, c, labels, mask); returns global tensors (no grad) + local offsets."""
        W, r = dist.get_world_size(), dist.get_rank()
        B, d = q.shape
        C = c.shape[0]
        nb_f = (B + C) * d * 4
        nb = nb_f + B * 8 + C
        nb_pad = (nb + 15) // 16 * 16
        send = torch.empty(nb_pad, dtype=torch.uint8, device=q.device)
        send[:B * d * 4].view(torch.float32).view(B, d).copy_(q.detach())
        send[B * d * 4:nb_f].view(torch.float32).view(C, d).copy_(c.detach())
        send[nb_f:nb_f + B * 8].view(torch.int64).copy_(labels)
        send[nb_f + B * 8:nb].copy_(mask.to(torch.uint8))
        recv = torch.empty(W, nb_pad, dtype=torch.uint8, device=q.device)
        dist.all_gather_into_tensor(recv.view(-1), send)
        q_all = recv[:, :B * d * 4].contiguous().view(torch.float32).view(W * B, d)
        c_all = recv[:, B * d * 4:nb_f].contiguous().view(torch.float32).view(W * C, d)
        lab = recv[:, nb_f:nb_f + B * 8].contiguous().view(torch.int64).view(W, B)
        lab = lab + (torch.arange(W, device=q.device, dtype=torch.int64) * C).unsqueeze(1)  # :189-190
        m_all = recv[:, nb_f + B * 8:nb].contiguous().view(W * C)
        return q_all, c_all, lab.reshape(-1), m_all, r * B, r * C

    def training_step(self, batch, batch_idx):
        query_ids = batch["query_ids"]
        contexts_ids = batch["contexts_ids"]
        dev = self.query_encoder.master.device
        pos_ctx_indices = batch["pos_ctx_indices"].to(dev, torch.int64)
        mask = batch["ctx_mask"].to(dev)
        query_repr, context_repr = self(query_ids, contexts_ids)
        pt = self.phase_timer
        if pt is not None:
            pt.mark("encoders_fwd")
        inv_t = 1.0 / float(self.softmax_temperature)
        pair_mask = None
        if self.in_batch_negatives:
            if self._is_ddp():
                q_all, c_all, labels, col_mask, q0, c0 = self._gather_global(query_repr, context_repr,
                                                                            pos_ctx_indices, mask)
                if pt is not None:
                    pt.mark("gather")
            else:
                q_all, c_all, labels = query_repr.detach(), context_repr.detach(), pos_ctx_indices
                col_mask, q0, c0 = mask.to(torch.uint8), 0, 0
        else:
            # only the contexts attached to each query are candidates (reference :199-207)
            Q, C = query_repr.shape[0], mask.shape[0]
            per = int(C / Q)
            cols = torch.arange(C, device=dev).unsqueeze(0)
            start = pos_ctx_indices.unsqueeze(1)
            inside = (cols >= start) & (cols < start + per)
            pair_mask = (~inside | mask.unsqueeze(0)).to(torch.uint8).contiguous()
            q_all, c_all, labels = query_repr.detach(), context_repr.detach(), pos_ctx_indices
            col_mask, q0, c0 = None, 0, 0
        loss = _ScoreCE.apply(query_repr, context_repr, q_all.contiguous(), c_all.contiguous(),
                              labels.contiguous(), None if col_mask is None else col_mask.contiguous(),
                              pair_mask, inv_t, q0, c0)
        if pt is not None:
            pt.mark("score_fwd")
        self.log("train_loss", loss, prog_bar=True)
        return loss

    # ------------------------------------------------------------------ evaluation
    def _eval_step(self, batch, batch_idx):
        dev = self.query_encoder.master.device
        pos_ctx_indices = batch["pos_ctx_indices"].to(dev, torch.int64)
        mask = batch["ctx_mask"].to(dev)
        query_repr, contexts_repr = self(batch["query_ids"], batch["contexts_ids"])
        loss_sum, _, scores, _ = ops.score_fwd(query_repr.contiguous(), contexts_repr.contiguous(),
                                               mask.to(torch.uint8).contiguous(), pos_ctx_indices, 1.0, True)
        loss = loss_sum[0] / query_repr.shape[0]
        return (self.compute_rank_metrics(scores, pos_ctx_indices), query_repr, contexts_repr, pos_ctx_indices,
                mask, loss)

    def compute_rank_metrics(self, pred_scores, target_labels):
        """(sum of ranks, sum of reciprocal ranks, hits@k) — one device-side pass instead of the reference's
        Python loop over a full sort (:235-246); rank = 1 + #scores strictly greater + #equal scores that a
        stable descending sort would place first (lower column index)."""
        labels = torch.as_tensor(target_labels, device=pred_scores.device, dtype=torch.int64)
        gold = pred_scores.gather(1, labels.unsqueeze(1))
        cols = torch.arange(pred_scores.shape[1], device=pred_scores.device).unsqueeze(0)
        ahead = (pred_scores > gold) | ((pred_scores == gold) & (cols < labels.unsqueeze(1)))
        pos = ahead.sum(1)
        rank = int((pos + 1).sum())
        mrr = float((1.0 / (pos + 1).double()).sum())
        score = int((pos < self.k).sum())
        return rank, mrr, score

    def _eval_epoch_end(self, outputs, log_prefix="valid"):
        total_avg_rank, total_ctx_count, total_count = 0, 0, 0
        total_mrr, total_loss, total_score = 0, 0, 0
        if self.in_batch_eval:
            for metrics, query_repr, contexts_repr, _, mask, loss in outputs:
                rank, mrr, score = metrics
                total_avg_rank += rank
                total_mrr += mrr
                total_score += score
                total_ctx_count += contexts_repr.size(0) - torch.sum(mask)
                total_count += query_repr.size(0)
                total_loss += loss
            total_ctx_count = total_ctx_count / len(outputs)
            total_loss = total_loss / len(outputs)
        else:
            qs, cs, ms, labels, offset = [], [], [], [], 0
            for _, query_repr, context_repr, target_labels, mask, _ in outputs:
                qs.append(query_repr)
                cs.append(context_repr)
                ms.append(mask)
                labels.append(target_labels + offset)
                offset += context_repr.size(0)
            all_c, all_m = torch.cat(cs, 0), torch.cat(ms, 0)
            labels = torch.cat(labels, 0)
            world = getattr(self.trainer, "world_size", 1) if self.trainer is not None else 1
            if world > 1:
                g_c, g_m = self.all_gather((all_c, all_m))
                labels = labels + g_c.size(1) * self.global_rank
                all_c = g_c.reshape(-1, g_c.shape[-1])
                all_m = g_m.reshape(-1)
            all_q = torch.cat(qs, 0)
            loss_sum, _, scores, _ = ops.score_fwd(all_q.contiguous(), all_c.contiguous(),
                                                   all_m.to(torch.uint8).contiguous(), labels.contiguous(), 1.0, True)
            total_count = all_q.size(0)
            total_ctx_count = scores.size(1) - torch.sum(all_m)
            total_avg_rank, total_mrr, total_score = self.compute_rank_metrics(scores, labels)
            total_loss = loss_sum[0] / total_count
        metrics = {
            log_prefix + "_avg_rank": total_avg_rank / total_count,
            log_prefix + "_mrr": total_mrr / total_count,
            log_prefix + f"_accuracy@{self.k}": total_score / total_count,
            log_prefix + "_ctx_count": total_ctx_count,
            log_prefix + "_loss": total_loss,
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
