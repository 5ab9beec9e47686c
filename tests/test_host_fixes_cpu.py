"""Host-side logic, all runnable without a GPU:
  * two live forwards of ONE encoder never share a save-for-backward workspace (shared_model=True aliasing);
  * a shared encoder hands its gradient slices to the all-reduce exactly once per step (last outstanding backward);
  * reference checkpoints written with transformers==3.4.0 (persistent `embeddings.position_ids`) load strictly;
  * val / test loaders shard like Lightning's DistributedSampler(shuffle=False);
  * world-2 gloo: `main.init_distributed`, log_dict(sync_dist=True), one checkpoint path for all ranks, the
    bf16-compressed (`fp16_grads`) gradient all-reduce, mean gradients for a plain torch optimizer.
"""
import os
import sys
import types

import torch
import torch.distributed as dist
import torch.multiprocessing as mp
from torch.utils.data import DistributedSampler

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TINY = dict(vocab_size=64, hidden_size=128, num_hidden_layers=2, num_attention_heads=2, intermediate_size=256,
            max_position_embeddings=40)


def test_workspace_pool_never_aliases_live_leases():
    from dpr_scale_b200.models.hf_model import _FwdState, _WorkspacePool
    pool = _WorkspacePool()
    dev = torch.device("cpu")
    a = pool.lease(1000, dev)
    b = pool.lease(1000, dev)                     # second live forward of the same shape (query + context pass)
    assert a.data_ptr() != b.data_ptr() and pool.leased == 2
    sa = _FwdState(None, None, None, a, pool)
    sa.release()
    sa.release()                                  # idempotent
    assert pool.leased == 1 and pool.idle is a
    c = pool.lease(500, dev)                      # an idle buffer that is large enough is reused ...
    assert c is a and pool.idle is None
    sb = _FwdState(None, None, None, b, pool)
    del sb                                        # ... and a dropped graph returns its lease through __del__
    assert pool.leased == 1 and pool.idle is b
    d = pool.lease(5000, dev)                     # too small: the idle buffer is dropped, a fresh one allocated
    assert d.numel() == 5000 and pool.idle is None
    pool.give_back(d)
    pool.give_back(c)
    assert pool.idle is d and pool.leased == 0    # only the largest idle buffer is kept


class _FakeEnc:
    """Stands in for HFEncoder behind the autograd glue: records which backward passes were allowed to sync."""

    def __init__(self):
        from dpr_scale_b200.models.hf_model import _FwdState
        self._FwdState = _FwdState
        self._pending_bwd = 0
        self.syncs = []
        self.last_dropout = (0.0, 0)

    def _run_forward(self, tokens, save, train_dropout=None, force_seed=None):
        n = tokens["input_ids"].shape[0]
        return torch.ones(n, 4), self._FwdState(None, None, None, None, None)

    def _run_backward(self, state, dpooled, sync=True):
        self.syncs.append(bool(sync))


def test_shared_encoder_syncs_gradients_once_per_step():
    from dpr_scale_b200.models.hf_model import _ChunkedEncoderFn, _EncoderFn
    enc = _FakeEnc()
    anchor = torch.zeros(1, requires_grad=True)
    tok = {"input_ids": torch.zeros(6, 3, dtype=torch.long)}
    # shared_model=True: query pass and context pass through the same encoder, one loss
    enc._pending_bwd += 1
    q = _EncoderFn.apply(anchor, enc, tok, True)
    enc._pending_bwd += 1
    c = _EncoderFn.apply(anchor, enc, tok, True)
    (q.sum() + c.sum()).backward()
    assert enc.syncs == [False, True] and enc._pending_bwd == 0
    # activation chunking: 6 sequences in chunks of 4 -> two backward chunks, only the last one may sync
    enc.syncs = []
    enc._pending_bwd += 1
    r = _ChunkedEncoderFn.apply(anchor, enc, tok, 4)
    r.sum().backward()
    assert enc.syncs == [False, True] and enc._pending_bwd == 0
    # shared + chunked: the first (chunked) backward must not sync at all
    enc.syncs = []
    enc._pending_bwd += 1
    a = _ChunkedEncoderFn.apply(anchor, enc, tok, 4)
    enc._pending_bwd += 1
    b = _EncoderFn.apply(anchor, enc, tok, True)
    (a.sum() + b.sum()).backward()
    assert sorted(enc.syncs) == [False, False, True] and enc.syncs[-1] is True


def test_reference_checkpoint_with_position_ids_buffer_loads_strictly():
    from dpr_scale_b200.models.hf_model import HFEncoder
    enc = HFEncoder.from_config(TINY, dropout=0.0)
    sd = {k: v.clone() for k, v in enc.state_dict().items()}
    want = sd["transformer.embeddings.word_embeddings.weight"] + 1.0
    sd["transformer.embeddings.word_embeddings.weight"] = want
    sd["transformer.embeddings.position_ids"] = torch.arange(40).unsqueeze(0)        # transformers==3.4.0 buffer
    enc.load_state_dict(sd)                                                            # strict
    assert torch.equal(enc.state_dict()["transformer.embeddings.word_embeddings.weight"], want)
    # and through the task (query_encoder.* / context_encoder.* prefixes, as Lightning checkpoints carry them)
    from dpr_scale_b200.task.dpr_task import DenseRetrieverTask
    task = DenseRetrieverTask(transform={}, datamodule=None, optim={}, shared_model=False,
                              model={"_target_": "dpr_scale_b200.models.hf_model.HFEncoder.from_config", "config": TINY})
    task.setup("fit")
    tsd = {k: v.clone() for k, v in task.state_dict().items()}
    for side in ("query_encoder", "context_encoder"):
        tsd[f"{side}.transformer.embeddings.position_ids"] = torch.arange(40).unsqueeze(0)
    task.load_state_dict(tsd)


def test_eval_order_is_lightnings_distributed_sampler():
    from dpr_scale_b200.datamodule.dpr import DenseRetrieverDataModuleBase
    for n in (1, 7, 10, 16):
        for world in (1, 2, 3, 4):
            for rank in range(world):
                dm = DenseRetrieverDataModuleBase.__new__(DenseRetrieverDataModuleBase)
                dm.datasets = {"valid": list(range(n))}
                dm.trainer = types.SimpleNamespace(world_size=world, global_rank=rank)
                want = list(DistributedSampler(range(n), num_replicas=world, rank=rank, shuffle=False)) if world > 1 \
                    else list(range(n))
                assert dm._eval_order("valid") == want, (n, world, rank)


class _StubEnc:
    """Arena-shaped stand-in: a flat fp32 gradient buffer the trainer reduces slice by slice."""

    def __init__(self, rank):
        self.grads = torch.arange(64, dtype=torch.float32) * (rank + 1) + 0.123
        self.master = torch.zeros(64)
        self.transformer = types.SimpleNamespace(_grads=self.grads, arena_params=lambda: [])


def _worker(rank, world, port, tmp, ret):
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), WORLD_SIZE=str(world), RANK=str(rank),
                      LOCAL_RANK=str(rank), DPRB_DIST_BACKEND="gloo")
    from dpr_scale_b200 import main as dmain
    assert dmain.init_distributed() == world and dist.is_initialized() and dist.get_world_size() == world
    out = {}
    # ---- log_dict(sync_dist=True): every rank ends up with the mean
    from dpr_scale_b200.utils.lightning_shim import LightningModule
    lm = LightningModule()
    d = {"valid_mrr": 0.25 + 0.5 * rank, "valid_loss": torch.tensor(2.0 + rank)}
    lm.log_dict(d, on_epoch=True, sync_dist=True)
    out["mrr"], out["loss"] = float(d["valid_mrr"]), float(d["valid_loss"])
    # ---- checkpoint: one path for everyone although only rank 0 can see the existing file
    from dpr_scale_b200.utils.checkpoint import ModelCheckpoint
    mydir = tmp if rank == 0 else os.path.join(tmp, "elsewhere")      # rank 1 probes a directory without the file
    os.makedirs(mydir, exist_ok=True)
    if rank == 0:
        open(os.path.join(tmp, "checkpoint_best.ckpt"), "w").close()
    dist.barrier()
    cb = ModelCheckpoint(dirpath=mydir, monitor="valid_mrr", mode="max", save_top_k=1, filename="checkpoint_best")
    cb.on_validation_end(torch.nn.Linear(2, 2), 0, 1, {"valid_mrr": out["mrr"]}, is_writer=rank == 0)
    out["best"] = cb.best_model_path
    # ---- gradient all-reduce: fp32 and bf16-compressed; every slice exactly once
    from dpr_scale_b200.trainer import Trainer
    tr = Trainer(max_steps=1, device="cpu")
    assert tr.world_size == world and tr.strategy is not None
    for compress in (False, True):
        enc = _StubEnc(rank)
        tr.task = types.SimpleNamespace(query_encoder=enc, context_encoder=enc, parameters=lambda: [])
        tr._pending = []
        tr.set_grad_compression(compress)
        tr._sync_slice(enc, 32, 64)
        tr._sync_slice(enc, 0, 32)
        tr._allreduce_grads()
        out[f"g{int(compress)}"] = enc.grads.clone()
    ret[rank] = out
    dist.barrier()
    dist.destroy_process_group()


def test_world2_gloo_host_logic(tmp_path):
    ret = mp.Manager().dict()
    mp.spawn(_worker, args=(2, 29643, str(tmp_path), ret), nprocs=2, join=True)
    a, b = ret[0], ret[1]
    assert abs(a["mrr"] - 0.5) < 1e-12 and abs(b["mrr"] - 0.5) < 1e-12 and a["loss"] == b["loss"] == 2.5
    assert a["best"] == b["best"] and a["best"].endswith("checkpoint_best-v1.ckpt")
    want = torch.arange(64, dtype=torch.float32) * 3 + 0.246
    assert torch.allclose(a["g0"], want, rtol=0, atol=1e-5) and torch.equal(a["g0"], b["g0"])
    # bf16 on the wire: 8 mantissa bits per addend
    assert torch.allclose(a["g1"], want, rtol=2 ** -7, atol=0) and torch.equal(a["g1"], b["g1"])
    assert not torch.equal(a["g1"], a["g0"])
