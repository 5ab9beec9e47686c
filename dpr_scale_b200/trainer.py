"""Mini trainer that speaks the Lightning hook names the task implements — used when pytorch_lightning is not
importable (it is absent from this image).  It covers what /root/reference/dpr_scale/main.py:32-50 asks of
``pytorch_lightning.Trainer`` for this path: ``fit`` (setup -> configure_optimizers -> loop of training_step /
backward / clip / optimizer + scheduler step), ``validate`` / ``test`` loops, one process per GPU with the
gradient all-reduce DDP would do — issued here as NCCL all-reduces over the encoders' FLAT gradient arenas,
chunked by layer range and overlapped with the remaining backward on a side stream.
"""
import os

import torch
import torch.distributed as dist

from . import ops
from .utils.lightning_shim import DDPStrategy


class Trainer:
    def __init__(self, max_steps=-1, max_epochs=1, gradient_clip_val=0.0, strategy=None, precision=16,
                 log_every_n_steps=50, limit_train_batches=None, limit_val_batches=None, device=None,
                 grad_bucket_layers=3, callbacks=None, check_val_every_n_epoch=1, **unused):
        self.max_steps = max_steps
        self.max_epochs = max_epochs
        self.gradient_clip_val = float(gradient_clip_val or 0.0)
        self.world_size = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        self.global_rank = dist.get_rank() if self.world_size > 1 else 0
        self.gpus = int(os.environ.get("LOCAL_WORLD_SIZE", self.world_size))   # GPUs of this node (sampler chunking)
        self.strategy = DDPStrategy() if (self.world_size > 1 or strategy in ("ddp", "ddp_sharded")) else None
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.datamodule = None
        self.global_step = 0
        self.grad_bucket_layers = grad_bucket_layers
        self.compress_grads = False
        self._comm_stream = None
        self.log_every_n_steps = log_every_n_steps
        self.limit_train_batches = limit_train_batches
        self.limit_val_batches = limit_val_batches
        self.weights_save_path = "."
        self.callbacks = list(callbacks or [])
        self.check_val_every_n_epoch = int(check_val_every_n_epoch or 0)
        self.current_epoch = 0

    def set_grad_compression(self, on):
        self.compress_grads = bool(on)

    # ------------------------------------------------------------------ setup
    def attach(self, task, datamodule=None, stage="fit"):
        self.datamodule = datamodule
        if datamodule is not None and hasattr(datamodule, "trainer"):
            datamodule.trainer = self
        task.trainer = self
        task.setup(stage)
        task.to(self.device)
        self.task = task
        if stage == "fit":
            opts, scheds = task.configure_optimizers()
            self.optimizer, self.scheduler = opts[0], scheds[0]["scheduler"]
            if hasattr(self.optimizer, "max_grad_norm"):
                self.optimizer.max_grad_norm = self.gradient_clip_val
                self.optimizer.grad_scale = 1.0 / self.world_size
            if hasattr(task, "on_pretrain_routine_start"):
                task.on_pretrain_routine_start()
            if self.world_size > 1:
                self._pending = []
                for e in self._encoders():
                    e.grad_sync = self._sync_slice
                    e.bwd_chunk_layers = self.grad_bucket_layers
        return task

    def _sync_slice(self, enc, lo, hi):
        """All-reduce (SUM) grads[lo:hi] of one encoder's flat arena as soon as backward has produced it; NCCL
        runs it on its own stream, ordered after the kernels enqueued so far, concurrently with the rest of backward.
        The encoder calls this only from the LAST outstanding backward over a slice (shared_model=True back-propagates
        twice into one arena), so every slice is reduced exactly once per step.
        `fp16_grads` (dpr_task.py:90-92, torch's fp16_compress_hook: cast -> all-reduce -> cast back) is the
        bf16-compressed form: half the bytes on the wire, fp32 arena before and after."""
        g = enc.grads[lo:hi]
        if self.compress_grads and g.is_cuda:
            h = torch.empty(hi - lo, dtype=torch.bfloat16, device=g.device)
            ops.cast_f32_bf16(g, h)
            self._pending.append((dist.all_reduce(h, async_op=True), g, h))
        elif self.compress_grads:
            h = g.to(torch.bfloat16)   # gloo / CPU tests of the host logic
            self._pending.append((dist.all_reduce(h, async_op=True), g, h))
        else:
            self._pending.append((dist.all_reduce(g, async_op=True), None, None))

    def _encoders(self):
        encs, seen = [], set()
        # a distillation task trains a query encoder only
        for e in (self.task.query_encoder, getattr(self.task, "context_encoder", self.task.query_encoder)):
            if id(e) not in seen:
                seen.add(id(e))
                encs.append(e)
        return encs

    # ------------------------------------------------------------------ one optimisation step
    def _allreduce_grads(self):
        """SUM all-reduce of the flat gradient arenas (the optimizer applies 1/world)."""
        if self.world_size <= 1:
            return
        for work, g, h in self._pending:  # issued chunk by chunk during backward (see _sync_slice)
            work.wait()
            if h is not None:
                ops.cast_bf16_f32(h, g) if g.is_cuda else g.copy_(h)
        self._pending = []
        extra = [p for p in self.task.parameters() if p.grad is not None and not self._in_arena(p)]
        for p in extra:
            dist.all_reduce(p.grad)

    def _in_arena(self, p):
        for e in self._encoders():
            m = e.master
            if m.data_ptr() <= p.data_ptr() < m.data_ptr() + m.numel() * 4:
                return True
        return False

    def training_step(self, batch, batch_idx=0):
        """zero_grad -> task.training_step -> backward -> grad all-reduce -> clip + AdamW -> LR schedule."""
        pt = getattr(self.task, "phase_timer", None)
        if pt is not None:
            pt.begin()
        self.optimizer.zero_grad()
        if pt is not None:
            pt.mark("zero_grad")
        loss = self.task.training_step(batch, batch_idx)
        loss.backward()
        if pt is not None:
            pt.mark("encoders_bwd")
        self._allreduce_grads()
        if pt is not None:
            pt.mark("grad_allreduce_exposed")
        if not hasattr(self.optimizer, "max_grad_norm"):
            # a plain torch optimizer: the SUM-reduced gradients become DDP's mean here, clipped or not
            if self.world_size > 1:
                done = set()
                for e in self._encoders():
                    if e.transformer._grads is not None:
                        e.transformer._grads.div_(self.world_size)
                        done.update(id(p) for _, p, _ in e.transformer.arena_params())
                for p in self.task.parameters():
                    if p.grad is not None and id(p) not in done:
                        p.grad.div_(self.world_size)
            if self.gradient_clip_val > 0:
                torch.nn.utils.clip_grad_norm_(self.task.parameters(), self.gradient_clip_val)
        self.optimizer.step()
        self.scheduler.step()
        self.global_step += 1
        if pt is not None:
            pt.mark("optimizer")
            pt.end()
        return loss

    # ------------------------------------------------------------------ loops
    def fit(self, task, datamodule=None):
        self.attach(task, datamodule, "fit")
        task.train()
        done = False
        for epoch in range(self.max_epochs if self.max_epochs and self.max_epochs > 0 else 10 ** 9):
            if hasattr(datamodule, "set_epoch"):
                datamodule.set_epoch(epoch)
            for i, batch in enumerate(datamodule.train_dataloader()):
                if self.limit_train_batches is not None and i >= self.limit_train_batches:
                    break
                loss = self.training_step(batch, i)
                if self.global_rank == 0 and self.global_step % self.log_every_n_steps == 0:
                    print(f"step {self.global_step} train_loss {float(loss):.4f}")
                if self.max_steps and 0 < self.max_steps <= self.global_step:
                    done = True
                    break
            self._end_of_epoch(task, datamodule, epoch)
            if done:
                break
        return task

    def _end_of_epoch(self, task, datamodule, epoch):
        """What Lightning does between epochs for this path: a validation pass, then the checkpoint callbacks
        (main.py:30-32 registers ModelCheckpoint monitoring valid_mrr)."""
        self.current_epoch = epoch
        metrics = None
        has_val = datamodule is not None and hasattr(datamodule, "val_dataloader")
        if has_val and self.check_val_every_n_epoch > 0 and (epoch + 1) % self.check_val_every_n_epoch == 0:
            metrics = self.validate(task, datamodule)
        for cb in self.callbacks:
            if hasattr(cb, "on_validation_end"):
                cb.on_validation_end(task, epoch, self.global_step, metrics, is_writer=self.global_rank == 0)
        if self.world_size > 1:
            dist.barrier()

    @torch.no_grad()
    def _eval_loop(self, task, loader, step_name, end_name, limit=None):
        task.eval()
        outs = []
        for i, batch in enumerate(loader):
            if limit is not None and i >= limit:
                break
            outs.append(getattr(task, step_name)(batch, i))
        res = getattr(task, end_name)(outs)
        task.train()
        return res

    def validate(self, task, datamodule=None):
        dm = datamodule or self.datamodule
        return self._eval_loop(task, dm.val_dataloader(), "validation_step", "validation_epoch_end", self.limit_val_batches)

    def test(self, task=None, datamodule=None, ckpt_path=None, **unused):
        task = task if task is not None else self.task
        dm = datamodule or self.datamodule
        if getattr(task, "trainer", None) is None:
            self.attach(task, dm, "test")
        if ckpt_path:                                   # "best" = the checkpoint callback's choice (main.py:46-47)
            from .utils.checkpoint import load_into
            if ckpt_path == "best":
                ckpt_path = next((cb.best_model_path for cb in self.callbacks if getattr(cb, "best_model_path", "")), "")
            if ckpt_path:
                load_into(task, ckpt_path)
                task.to(self.device)
        return self._eval_loop(task, dm.test_dataloader(), "test_step", "test_epoch_end")
