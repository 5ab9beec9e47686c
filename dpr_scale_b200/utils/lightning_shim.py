"""Minimal stand-ins for the pytorch_lightning symbols the task uses, used ONLY when Lightning is not
importable (it is absent from this image and cannot be installed).  When the real library is present the
task subclasses the real ``LightningModule`` instead.

Mirrors the surface used at /root/reference/dpr_scale/task/dpr_task.py:8-9,36,165,174,213,310:
``LightningModule.{save_hyperparameters, log, log_dict, all_gather, global_rank, trainer}`` and the
``DDPStrategy`` / ``DDPShardedStrategy`` marker classes.  ``all_gather`` follows PL 1.6.4 semantics: per
tensor ``dist.all_gather`` -> ``torch.stack(dim=0)`` without gradient; identity when not distributed.
"""
import inspect

import torch
import torch.distributed as dist
import torch.nn as nn

try:  # pragma: no cover - exercised only where Lightning exists
    from pytorch_lightning import LightningDataModule, LightningModule  # type: ignore
    from pytorch_lightning.strategies import DDPShardedStrategy, DDPStrategy  # type: ignore
    HAVE_LIGHTNING = True
except Exception:  # noqa
    HAVE_LIGHTNING = False

    class DDPStrategy:  # marker: "one process per GPU, gradients all-reduced"
        pass

    class DDPShardedStrategy(DDPStrategy):
        pass

    class LightningDataModule:
        def __init__(self):
            self.trainer = None

    class LightningModule(nn.Module):
        def __init__(self):
            super().__init__()
            self.trainer = None
            self.logged = {}
            self.hparams = {}

        def save_hyperparameters(self):
            frame = inspect.currentframe().f_back
            args = inspect.getargvalues(frame)
            self.hparams = {k: args.locals[k] for k in args.args if k != "self"}
            if args.keywords and args.keywords in args.locals:
                self.hparams.update(args.locals[args.keywords])

        def log(self, name, value, **kwargs):
            self.logged[name] = value

        def log_dict(self, d, sync_dist=False, **kwargs):
            # Lightning's sync_dist=True reduces every logged value with a mean over the ranks, so that rank-level
            # callbacks (ModelCheckpoint's monitor) see ONE number.  Values are reduced in place in `d`.
            if sync_dist and dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
                keys = sorted(d)
                dev = None
                for k in keys:
                    if torch.is_tensor(d[k]) and d[k].is_cuda:
                        dev = d[k].device
                if dev is None and dist.get_backend() == "nccl":
                    dev = torch.device("cuda", torch.cuda.current_device())
                vals = torch.tensor([float(d[k]) for k in keys], dtype=torch.float64, device=dev)
                dist.all_reduce(vals)
                vals /= dist.get_world_size()
                for k, v in zip(keys, vals.tolist()):
                    d[k] = v
            self.logged.update(d)

        @classmethod
        def load_from_checkpoint(cls, checkpoint_path, map_location=None, **kwargs):
            """Rebuild the task from a checkpoint's ``hyper_parameters`` (kwargs override them), build its modules
            through ``on_load_checkpoint`` and load the ``state_dict`` strictly - Lightning's classmethod of that name
            for the files utils/checkpoint.ModelCheckpoint writes."""
            ckpt = torch.load(checkpoint_path, map_location="cpu", weights_only=False)
            if not isinstance(ckpt, dict) or "state_dict" not in ckpt:
                raise ValueError(f"{checkpoint_path} is not a checkpoint: it has no state_dict")
            hparams = dict(ckpt.get("hyper_parameters") or {})
            hparams.update(kwargs)
            model = cls(**hparams)
            if hasattr(model, "on_load_checkpoint"):
                model.on_load_checkpoint(ckpt)
            model.load_state_dict(ckpt["state_dict"])
            return model.to(map_location) if map_location is not None else model

        @property
        def global_rank(self):
            return dist.get_rank() if dist.is_available() and dist.is_initialized() else 0

        def all_gather(self, data, group=None, sync_grads=False):
            def one(t):
                if not (dist.is_available() and dist.is_initialized()):
                    return t
                with torch.no_grad():
                    src = t.to(torch.uint8) if t.dtype == torch.bool else t
                    outs = [torch.zeros_like(src) for _ in range(dist.get_world_size())]
                    dist.all_gather(outs, src.contiguous(), group=group)
                    res = torch.stack(outs, dim=0)
                    return res.to(torch.bool) if t.dtype == torch.bool else res
            if isinstance(data, (tuple, list)):
                return type(data)(one(t) for t in data)
            return one(data)
