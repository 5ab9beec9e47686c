"""2-rank NCCL parity of the global in-batch-negative path (configs[2]) against the 2-rank golden produced by the
unmodified reference under gloo: every rank reports the reference's loss; after the trainer's gradient all-reduce
(SUM, scaled 1/W by the optimizer) the flat gradient equals the mean of the reference's per-rank gradients."""
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _worker(rank, world, port, ret):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    from dpr_scale_b200.task.dpr_task import DenseRetrieverTask
    from dpr_scale_b200.trainer import Trainer
    from tests.test_task_gpu import CFG, _batch
    from tests.util import load_golden, sub
    g2, g1 = load_golden("golden_2rank.npz"), load_golden("golden_1rank.npz")
    task = DenseRetrieverTask(transform={}, datamodule=None, shared_model=False, softmax_temperature=float(g1["temperature"]),
                              model={"_target_": "dpr_scale_b200.models.hf_model.HFEncoder.from_config", "config": CFG, "dropout": 0.0},
                              optim={"_target_": "dpr_scale_b200.optim.FusedAdamW", "lr": 0.0})
    tr = Trainer(max_steps=10, gradient_clip_val=0.0, device=torch.device("cuda", rank), grad_bucket_layers=1)
    tr.attach(task, None, "fit")
    task.query_encoder.load_state_dict(sub(g1, "sd_q/"))
    task.context_encoder.load_state_dict(sub(g1, "sd_c/"))
    task.train()
    batch = _batch(g2, f"rank{rank}/batch/")
    tr.optimizer.zero_grad()
    loss = task.training_step(batch, 0)
    loss.backward()
    tr._allreduce_grads()
    torch.cuda.synchronize()
    num = den = 0.0
    for name, enc in (("q", task.query_encoder), ("c", task.context_encoder)):
        r0, r1 = sub(g2, f"rank0/grad_{name}/"), sub(g2, f"rank1/grad_{name}/")
        for k, p in enc.named_parameters():
            if k not in r0:
                continue
            want = r0[k] + r1[k]  # SUM over ranks (the optimizer applies 1/W)
            got = p.grad.detach().float().cpu()
            num += float(((got - want).double() ** 2).sum())
            den += float((want.double() ** 2).sum())
    ret[rank] = (float(loss), float(g2[f"rank{rank}/loss"]), (num / den) ** 0.5, float(g1["amp_global_rel"]))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_global_negatives_match_reference():
    import torch.multiprocessing as mp
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(2, 29655, ret), nprocs=2, join=True)
    for r in (0, 1):
        loss, want, grel, amp = ret[r]
        assert abs(loss - want) <= 5e-2, (loss, want)
        assert grel <= 1.5 * amp, (grel, amp)
    assert abs(ret[0][0] - ret[1][0]) < 1e-6  # every rank computes the same global loss


def _shared_worker(rank, world, port, ret):
    """shared_model=True (the reference's constructor default) on 2 ranks: ONE encoder back-propagates twice per step into
    one gradient arena; the bucketed all-reduce must reduce every slice exactly once.
    Reference semantics (dpr_task.py:163-195 + DDP): SUM over ranks of the per-rank gradients == gradient of the global
    loss, i.e. what ONE process computes on the concatenated batch."""
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    from dpr_scale_b200.task.dpr_task import DenseRetrieverTask
    from dpr_scale_b200.trainer import Trainer
    from tests.test_task_gpu import CFG, _batch
    from tests.util import load_golden, rel_l2, sub
    g2, g1 = load_golden("golden_2rank.npz"), load_golden("golden_1rank.npz")
    T = float(g1["temperature"])

    def make(distributed):
        task = DenseRetrieverTask(transform={}, datamodule=None, shared_model=True, softmax_temperature=T,
                                  model={"_target_": "dpr_scale_b200.models.hf_model.HFEncoder.from_config", "config": CFG,
                                         "dropout": 0.0},
                                  optim={"_target_": "dpr_scale_b200.optim.FusedAdamW", "lr": 0.0})
        tr = Trainer(max_steps=10, gradient_clip_val=0.0, device=torch.device("cuda", rank), grad_bucket_layers=1)
        if not distributed:
            tr.world_size, tr.strategy = 1, None
        tr.attach(task, None, "fit")
        task.query_encoder.load_state_dict(sub(g1, "sd_q/"))
        task.train()
        return task, tr

    task, tr = make(True)
    assert task.query_encoder is task.context_encoder
    batches = [_batch(g2, f"rank{r}/batch/") for r in range(world)]
    tr.optimizer.zero_grad()
    loss = task.training_step(batches[rank], 0)
    loss.backward()
    tr._allreduce_grads()
    torch.cuda.synchronize()
    got = task.query_encoder.grads.clone()
    rel = -1.0
    if rank == 0:
        # single-process reference on the concatenated global batch (queries and contexts padded to a common length)
        ref, rtr = make(False)
        rtr.task.trainer = None

        def cat(key):
            parts = [b[key] for b in batches]
            S = max(p["input_ids"].shape[1] for p in parts)
            out = {}
            for k in parts[0]:
                out[k] = torch.cat([torch.nn.functional.pad(p[k], (0, S - p[k].shape[1])) for p in parts], 0)
            return out
        C = batches[0]["contexts_ids"]["input_ids"].shape[0]
        big = {"query_ids": cat("query_ids"), "contexts_ids": cat("contexts_ids"),
               "pos_ctx_indices": torch.cat([b["pos_ctx_indices"] + i * C for i, b in enumerate(batches)]),
               "ctx_mask": torch.cat([b["ctx_mask"] for b in batches])}
        ref.query_encoder.zero_grad()
        rloss = ref.training_step(big, 0)
        rloss.backward()
        torch.cuda.synchronize()
        rel = rel_l2(got, ref.query_encoder.grads)
        ret["loss"] = (float(loss), float(rloss))
    ret[rank] = rel
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_shared_model_gradients_reduced_once():
    import torch.multiprocessing as mp
    ret = mp.Manager().dict()
    mp.spawn(_shared_worker, args=(2, 29657, ret), nprocs=2, join=True)
    loss, rloss = ret["loss"]
    assert abs(loss - rloss) <= 2e-3, (loss, rloss)
    # the double all-reduce gave W * sum_ctx + sum_q: a relative error of order 1; bf16 / atomics noise is ~1e-2
    assert 0 <= ret[0] <= 3e-2, ret[0]
