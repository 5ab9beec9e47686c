#!/usr/bin/env python3
"""bench.py — query+ctx pairs/sec of the bi-encoder contrastive training step (BASELINE.json metric).

  python bench.py --gpus N --steps K --warmup W            # this repo's sm_90a path (one rank per GPU)
  python bench.py ... --dump-outputs DIR                   # also write what the last timed step computed (.npy)
  python bench.py --impl reference ...                      # the reference's own CPU path (HF + torch, fp32)
  python bench.py --impl stock ...                          # stock HF + PyTorch on the same GPU (the 1.5x denominator)

The default line also carries: `stock_gpu` / `vs_stock` (stock HF + PyTorch on the SAME GPU right after our arm -
the denominator of north_star's 1.5x target), `phases` (CUDA-event time per phase of the step), `selfcheck` (N > 1:
NCCL parity against the reference-generated goldens before timing) and, at N > 1, `grad_allreduce_bf16` (the same step
with the `fp16_grads` compressed gradient all-reduce).

A "step" = zero_grad -> both encoders fwd -> (all-gather) -> fused scoring+CE -> backward -> (grad all-reduce)
-> clip(2.0) + AdamW + LambdaLR, on one synthetic batch of configs[1]/[2]: BERT-base, S=128, 128 queries/GPU,
1 pos + 7 hard negatives (1024 contexts/GPU), in-batch (global when N>1) negatives.  Prints ONE JSON line.
"""
import argparse
import contextlib
import ctypes
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

BERT_BASE = dict(model_type="bert", vocab_size=30522, hidden_size=768, num_hidden_layers=12, num_attention_heads=12,
                 intermediate_size=3072, max_position_embeddings=512, type_vocab_size=2, layer_norm_eps=1e-12,
                 pad_token_id=0, initializer_range=0.02)
ROBERTA_LARGE = dict(model_type="roberta", vocab_size=50265, hidden_size=1024, num_hidden_layers=24,
                     num_attention_heads=16, intermediate_size=4096, max_position_embeddings=514, type_vocab_size=1,
                     layer_norm_eps=1e-5, pad_token_id=1, initializer_range=0.02)
WORKLOADS = {
    # name: (model cfg, queries/GPU, hard negs, seq len)
    "bert-base_s128_b128_n7": (BERT_BASE, 128, 7, 128),          # BASELINE configs[1] / [2]  (the headline)
    "bert-base_s64_b8_n1": (BERT_BASE, 8, 1, 64),                # configs[0] shape
    "roberta-large_s256_b16_n15": (ROBERTA_LARGE, 16, 15, 256),  # configs[3]'s model and recipe at an 80 GB batch
}
# RoBERTa-large runs with LEAN activations (22 KB instead of 32 KB per token and layer; gelu / gelu' / attention output
# rebuilt in backward): 69 632 tokens x 24 layers per GPU then fit an 80 GB H100 without recomputing the forward.
# --act-chunk N selects the older chunked-recompute path.
ACT_CHUNK = {}
LEAN = {"roberta-large_s256_b16_n15"}


def flops_per_token_train(cfg, S):
    H, I, L = cfg["hidden_size"], cfg["intermediate_size"], cfg["num_hidden_layers"]
    return 3 * L * (2 * (4 * H * H + 2 * H * I) + 4 * S * H)  # fwd + bwd = 3 x fwd: QKV / out / FFN GEMMs + QK^T and PV


def synth_batch(rank, cfg, B, n, S, pin=True):
    """Benchmark inputs, variant A: all sequences exactly S tokens, mask all ones."""
    g = torch.Generator().manual_seed(1234 + rank)
    C = B * (1 + n)

    def toks(N):
        ids = torch.randint(1000, 30000, (N, S), generator=g)
        ids[:, 0] = 101
        ids[:, -1] = 102
        d = {"input_ids": ids, "token_type_ids": torch.zeros_like(ids), "attention_mask": torch.ones_like(ids)}
        return {k: (v.pin_memory() if pin else v) for k, v in d.items()}

    b = {"query_ids": toks(B), "contexts_ids": toks(C), "pos_ctx_indices": torch.arange(B) * (1 + n),
         "ctx_mask": torch.zeros(C, dtype=torch.bool)}
    if pin:
        b["pos_ctx_indices"] = b["pos_ctx_indices"].pin_memory()
        b["ctx_mask"] = b["ctx_mask"].pin_memory()
    return b


def to_device(batch, dev):
    out = {}
    for k, v in batch.items():
        out[k] = {kk: vv.to(dev, non_blocking=True) for kk, vv in v.items()} if isinstance(v, dict) else v.to(dev, non_blocking=True)
    return out


def batch_bytes(batch):
    n = 0
    for v in batch.values():
        for t in (v.values() if isinstance(v, dict) else [v]):
            n += t.numel() * t.element_size()
    return n


class ClockSampler:
    """nvidia-smi clocks / throttle reasons sampled every 200 ms during the timed region."""
    Q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, index):
        self.index, self.rows, self.proc = index, [], None

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.index), "--query-gpu=" + self.Q,
                                          "--format=csv,noheader,nounits", "-lms", "200"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            threading.Thread(target=self._read, daemon=True).start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([x.strip() for x in line.split(",")])

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        sm, mx, reasons = [], None, set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for r in self.rows:
            try:
                sm.append(float(r[0]))
                mx = float(r[1])
                for nm, val in zip(names, r[3:7]):
                    if val.lower().startswith("active"):
                        reasons.add(nm)
            except Exception:
                pass
        sm.sort()
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": mx, "reasons": sorted(reasons),
                "samples": len(sm)}


def usable_cores():
    """Host threads this process may really use: affinity mask, capped by the cgroup CPU quota (shared GPU boxes
    report 128 logical CPUs but throttle the container), and by 32 (HF BERT at these sample sizes does not scale further)."""
    try:
        n = len(os.sched_getaffinity(0))
    except Exception:
        n = os.cpu_count() or 1
    try:
        with open("/sys/fs/cgroup/cpu.max") as f:
            quota, period = f.read().split()
        if quota != "max":
            n = min(n, max(1, int(float(quota) / float(period))))
    except Exception:
        pass
    return max(1, min(n, 32))


def peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return d.get("bf16_tflops_sustained", 989.0), d.get("hbm_gbs", 3350.0), "measured (MEASURED_PEAKS.json, sustained)"
    return 989.0, 3350.0, "H100 SXM data sheet (dense bf16, HBM3)"


# --------------------------------------------------------------------------------------- CPU reference path
REF_ROOT = "/root/reference"


def reference_encoders(cfg, dropout):
    """(query encoder, context encoder, kind) of the reference path.
    kind == "reference": the UNMODIFIED /root/reference/dpr_scale/models/hf_model.py:HFEncoder, imported as is and
    instantiated from a temp `save_pretrained` directory - only possible where /root/reference exists (the authoring
    container).  kind == "port": oracle/hf_path.CLSEncoder, the same arithmetic (HF AutoModel + CLS pooling) without
    the reference tree - what the GPU box runs, because a Python reference cannot travel and its sources may not be
    copied into the repo."""
    from oracle import hf_path
    hf_cfg = hf_path.make_config(cfg["model_type"], **{k: v for k, v in cfg.items() if k not in ("model_type",)})
    torch.manual_seed(0)
    if os.path.exists(os.path.join(REF_ROOT, "dpr_scale", "models", "hf_model.py")) and not os.environ.get("DPRB_REF_PORT"):
        import shutil
        import tempfile
        from transformers import AutoModel
        hf_cfg.attention_probs_dropout_prob = hf_cfg.hidden_dropout_prob = dropout
        d = tempfile.mkdtemp(prefix="dprb_ref_")
        try:
            AutoModel.from_config(hf_cfg).save_pretrained(d)
            sys.path.insert(0, REF_ROOT)
            from dpr_scale.models.hf_model import HFEncoder as RefEncoder
            with contextlib.redirect_stdout(sys.stderr), contextlib.redirect_stderr(open(os.devnull, "w")):
                q, c = RefEncoder(model_path=d, dropout=dropout), RefEncoder(model_path=d, dropout=dropout)
            return q, c, "reference"
        finally:
            shutil.rmtree(d, ignore_errors=True)
    return hf_path.CLSEncoder(hf_cfg, dropout=dropout), hf_path.CLSEncoder(hf_cfg, dropout=dropout), "port"


def cpu_reference_step_factory(cfg, pairs, n, S, threads):
    """The reference's own CPU path: HFEncoder x2 (fp32) + reference scoring/CE + clip + torch AdamW."""
    from oracle import task as otask
    torch.set_num_threads(threads)
    qe, ce, kind = reference_encoders(cfg, 0.1)
    cpu_reference_step_factory.kind = kind
    params = [p for p in list(qe.parameters()) + list(ce.parameters())]
    opt = torch.optim.AdamW(params, lr=1e-5, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0)
    batch = synth_batch(0, cfg, pairs, n, S, pin=False)

    def step():
        opt.zero_grad()
        q, c = qe(batch["query_ids"]), ce(batch["contexts_ids"])
        loss, _ = otask.in_batch_loss(q, c, batch["ctx_mask"], batch["pos_ctx_indices"], 1.0)
        loss.backward()
        torch.nn.utils.clip_grad_norm_([p for p in params if p.grad is not None], 2.0)
        opt.step()
        return float(loss)
    return step


def time_cpu_reference(cfg, pairs, n, S, steps, warmup, threads):
    step = cpu_reference_step_factory(cfg, pairs, n, S, threads)
    for _ in range(warmup):
        step()
    t0 = time.perf_counter()
    for _ in range(steps):
        step()
    dt = time.perf_counter() - t0
    return pairs * steps / dt, dt / steps, cpu_reference_step_factory.kind


# --------------------------------------------------------------------------------------- main arms
def run_reference(args, workload):
    cfg, B, n, S = WORKLOADS[workload]
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    threads = usable_cores()
    pairs = args.ref_pairs  # bounded sample of the same workload: `pairs` queries with 1+n contexts each, S tokens
    steps, warmup = args.steps, args.warmup
    value, spstep, kind = time_cpu_reference(cfg, pairs, n, S, steps, warmup, threads)
    line = {
        "impl": "reference", "metric": "query+ctx pairs/sec (BERT-base, seq128)", "value": value, "unit": "pairs/s",
        "n_gpus": args.gpus, "steps": steps, "warmup": warmup, "ms_per_step": spstep * 1e3, "higher_is_better": True,
        "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": workload, "sample_pairs_per_step": pairs, "hard_negatives": n, "seq_len": S,
                   "dropout": 0.1, "optimizer": "torch.optim.AdamW + clip 2.0"},
        "cpu_baseline": {"value": value, "unit": "pairs/s", "cores": threads, "kind": kind,
                         "sample": f"{pairs} pairs/step x {steps} steps of {workload} "
                                   f"({'unmodified reference HFEncoder' if kind == 'reference' else 'HF AutoModel + CLS pooling (port: /root/reference is absent on this box)'}"
                                   f" x2 fp32, fwd+bwd+clip+AdamW)"},
        "e2e": {"value": value, "unit": "pairs/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0,
    }
    print(json.dumps(line))


def time_stock(cfg, B, n, S, dropout, dtype, steps, warmup, dev, sample_clocks=True):
    """Stock HF + PyTorch on the GPU - the denominator of north_star's 1.5x: the reference's encoder class (see
    reference_encoders) x2, reference scoring / CE, torch.optim.AdamW(fused), clip_grad_norm_(2.0), under
    torch.autocast fp16 + GradScaler (= the reference's `precision: 16`, conf/trainer/slurm.yaml:15) or bf16; default
    SDPA attention; batch pre-staged on the device; CUDA events."""
    from oracle import task as otask
    qe, ce, kind = reference_encoders(cfg, dropout)
    qe, ce = qe.to(dev).train(), ce.to(dev).train()
    params = list(qe.parameters()) + list(ce.parameters())
    opt = torch.optim.AdamW(params, lr=1e-5, fused=True)
    batch = to_device(synth_batch(0, cfg, B, n, S), dev)
    amp = torch.bfloat16 if dtype == "bf16" else torch.float16
    scaler = torch.amp.GradScaler("cuda", enabled=(amp == torch.float16))

    def step():
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=amp):
            q, c = qe(batch["query_ids"]), ce(batch["contexts_ids"])
            loss, _ = otask.in_batch_loss(q, c, batch["ctx_mask"], batch["pos_ctx_indices"], 1.0)
        scaler.scale(loss).backward()
        scaler.unscale_(opt)
        torch.nn.utils.clip_grad_norm_([p for p in params if p.grad is not None], 2.0)
        scaler.step(opt)
        scaler.update()
        return loss

    torch.cuda.reset_peak_memory_stats(dev)
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    sampler = ClockSampler(dev.index or 0)
    if sample_clocks:
        sampler.start()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    clocks = sampler.stop() if sample_clocks else None
    ms = e0.elapsed_time(e1) / steps
    out = {"value": B / (ms / 1e3), "unit": "pairs/s", "ms_per_step": ms, "dtype": dtype, "steps": steps,
           "warmup": warmup, "encoder": kind, "attn": "sdpa", "dropout": dropout,
           "optimizer": "torch.optim.AdamW(fused) + clip_grad_norm_ 2.0" + (" + GradScaler" if dtype == "fp16" else ""),
           "peak_mem_gb": torch.cuda.max_memory_allocated(dev) / 2 ** 30, "clocks": clocks}
    del qe, ce, params, opt, batch
    import gc
    gc.collect()
    torch.cuda.empty_cache()
    return out


def run_stock(args, workload):
    cfg, B, n, S = WORKLOADS[workload]
    dev = torch.device("cuda", 0)
    r = time_stock(cfg, B, n, S, args.dropout, args.stock_dtype, args.steps, args.warmup, dev)
    r.update({"impl": "stock", "metric": "query+ctx pairs/sec (BERT-base, seq128)", "n_gpus": 1, "data": "synthetic",
              "higher_is_better": True, "config": {"workload": workload}})
    print(json.dumps(r))


# --------------------------------------------------------------------------------------- multi-GPU self-check
TINY_CFG = dict(vocab_size=64, hidden_size=128, num_hidden_layers=2, num_attention_heads=2, intermediate_size=256,
                max_position_embeddings=40)


def selfcheck(world, rank, dev):
    """NCCL parity BEFORE timing (the 1-GPU test box skips the NCCL pytest): the tiny golden model, one rank-specific
    batch per rank, global in-batch negatives through the packed all-gather, backward, the trainer's gradient
    all-reduce - against vectors the UNMODIFIED reference produced under gloo at the same world size
    (tests/golden/make_golden.py: per-rank loss; sum over ranks of every parameter gradient).  Golden files only: no
    oracle code runs here.  Gates: |loss - reference| <= 5e-2; global gradient rel-L2 <= 1.5x the reference's own
    bf16-autocast deviation (recorded in golden_1rank.npz)."""
    import numpy as np
    from dpr_scale_b200.task.dpr_task import DenseRetrieverTask
    from dpr_scale_b200.trainer import Trainer
    gdir = os.path.join(ROOT, "tests", "golden")
    name = {2: "golden_2rank.npz", 4: "golden_world4.npz", 8: "golden_world8.npz"}.get(world)
    if name is None or not os.path.exists(os.path.join(gdir, name)):
        return {"skipped": f"no reference golden for world size {world}"}
    z, g1 = np.load(os.path.join(gdir, name)), np.load(os.path.join(gdir, "golden_1rank.npz"))
    T = float(g1["temperature"])
    task = DenseRetrieverTask(transform={}, datamodule=None, shared_model=False, softmax_temperature=T,
                              model={"_target_": "dpr_scale_b200.models.hf_model.HFEncoder.from_config",
                                     "config": TINY_CFG, "dropout": 0.0},
                              optim={"_target_": "dpr_scale_b200.optim.FusedAdamW", "lr": 0.0})
    tr = Trainer(max_steps=10, gradient_clip_val=0.0, device=dev, grad_bucket_layers=1)
    with contextlib.redirect_stdout(sys.stderr):
        tr.attach(task, None, "fit")
    for side, enc in (("q", task.query_encoder), ("c", task.context_encoder)):
        pre = f"sd_{side}/"
        enc.load_state_dict({k[len(pre):]: torch.from_numpy(g1[k]) for k in g1.files if k.startswith(pre)})
    task.train()
    pre = f"rank{rank}/batch/"
    flat = {k[len(pre):]: torch.from_numpy(z[k]) for k in z.files if k.startswith(pre)}
    batch = {"query_ids": {k[len("query_ids/"):]: v for k, v in flat.items() if k.startswith("query_ids/")},
             "contexts_ids": {k[len("contexts_ids/"):]: v for k, v in flat.items() if k.startswith("contexts_ids/")},
             "pos_ctx_indices": flat["pos_ctx_indices"], "ctx_mask": flat["ctx_mask"].bool()}
    tr.optimizer.zero_grad()
    loss = task.training_step(batch, 0)
    loss.backward()
    tr._allreduce_grads()
    torch.cuda.synchronize()
    num = den = 0.0
    for side, enc in (("q", task.query_encoder), ("c", task.context_encoder)):
        for k, p in enc.named_parameters():
            if world == 2:
                a, b = f"rank0/grad_{side}/{k}", f"rank1/grad_{side}/{k}"
                if a not in z.files:
                    continue
                want = torch.from_numpy(z[a]) + torch.from_numpy(z[b])
            else:
                a = f"gradsum_{side}/{k}"
                if a not in z.files:
                    continue
                want = torch.from_numpy(z[a])
            got = p.grad.detach().float().cpu()
            num += float(((got - want).double() ** 2).sum())
            den += float((want.double() ** 2).sum())
    res = torch.tensor([abs(float(loss) - float(z[f"rank{rank}/loss"])), (num / den) ** 0.5], device=dev,
                       dtype=torch.float64)
    dist.all_reduce(res, op=dist.ReduceOp.MAX)
    amp = float(g1["amp_global_rel"])
    loss_err, grad_rel = float(res[0]), float(res[1])
    del task, tr
    return {"ok": bool(loss_err <= 5e-2 and grad_rel <= 1.5 * amp), "world": world, "golden": "tests/golden/" + name,
            "max_loss_err": loss_err, "max_grad_rel_l2": grad_rel, "gate_grad_rel_l2": 1.5 * amp, "gate_loss": 5e-2,
            "what": "tiny golden model, per-rank batches, packed all-gather + fused scoring + backward + gradient "
                    "all-reduce over NCCL vs the unmodified reference under gloo at the same world size"}


def dataloader_leg(trainer, dev, B, n, S, steps, warmup):
    """One end-to-end number including the dataloader.  A synthetic DPR-format JSONL (texts long
    enough that every sequence truncates to exactly S tokens, i.e. the named shape) goes through the repo's input
    pipeline - mmap line index, JSON + negative sampling, tokenisation, pinned staging, side-stream H2D - while the GPU
    trains; the loss is read back every step.  Returns (ms per step, rows per batch)."""
    import shutil
    import tempfile

    import numpy as np
    from transformers import BertConfig

    from dpr_scale_b200.datamodule.dpr import DenseRetrieverJsonlDataModule
    from dpr_scale_b200.transforms.hf_transform import HFTransform
    tmp = tempfile.mkdtemp(prefix="dprb_bench_")
    try:
        words = np.array(["w%05d" % i for i in range(30000)])
        with open(os.path.join(tmp, "vocab.txt"), "w") as f:
            f.write("\n".join(["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"] + words.tolist()) + "\n")
        BertConfig(vocab_size=30005).save_pretrained(tmp)
        rng = np.random.RandomState(0)
        rows = B * (steps + warmup + 1)
        path = os.path.join(tmp, "train.jsonl")
        with open(path, "w") as f:
            for r in range(rows):
                w = words[rng.randint(0, 30000, size=(n + 3, S + 16))]
                ctxs = [{"title": "", "text": " ".join(w[j]), "passage_id": str(r * 100 + j)} for j in range(n + 2)]
                f.write(json.dumps({"question": " ".join(w[n + 2]), "positive_ctxs": ctxs[:1], "negative_ctxs": [],
                                    "hard_negative_ctxs": ctxs[1:]}) + "\n")
        dm = DenseRetrieverJsonlDataModule(transform=HFTransform(model_path=tmp, max_seq_len=S), train_path=path,
                                           val_path=path, test_path=path, batch_size=B, num_negative=n,
                                           prefetch_batches=4, device_prefetch=True)
        dm.trainer = trainer
        it = iter(dm.train_dataloader())
        for i in range(warmup + 1):
            b = next(it)
            float(trainer.training_step(b, i))
        assert tuple(b["contexts_ids"]["input_ids"].shape) == (B * (1 + n), S), b["contexts_ids"]["input_ids"].shape
        assert tuple(b["query_ids"]["input_ids"].shape) == (B, S)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        host = torch.empty(steps, dtype=torch.float32).pin_memory()
        ready = [torch.cuda.Event() for _ in range(steps)]
        e0.record()
        for i in range(steps):               # loss of step i read while step i+1 runs, as in the e2e leg
            loss = trainer.training_step(next(it), i)
            host[i:i + 1].copy_(loss.detach().reshape(1), non_blocking=True)
            ready[i].record()
            if i > 0:
                ready[i - 1].synchronize()
                float(host[i - 1])
        ready[steps - 1].synchronize()
        float(host[steps - 1])
        e1.record()
        torch.cuda.synchronize()
        it.close()
        return e0.elapsed_time(e1) / steps
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


DUMP_SAMPLE = 1 << 21   # parameters sampled per encoder (8 MB of float32 each)


def dump_outputs(out_dir, loss, task):
    """What the last timed training step left to its caller: the loss it returned and the parameters its optimizer step
    wrote (both encoders; a fixed, seeded sample of each flat parameter vector, the same indices in every run).  The
    pooler, which the CLS-pooled path never reads, is left out."""
    import numpy as np
    torch.cuda.synchronize()
    os.makedirs(out_dir, exist_ok=True)
    np.save(os.path.join(out_dir, "loss.npy"), np.array([float(loss)], dtype=np.float64))
    for name, enc in (("query_encoder", task.query_encoder), ("context_encoder", task.context_encoder)):
        flat = torch.cat([p.detach().reshape(-1).float() for n, p in enc.named_parameters() if ".pooler." not in n])
        g = torch.Generator().manual_seed(2024)
        idx = torch.randperm(flat.numel(), generator=g)[:DUMP_SAMPLE].sort().values
        np.save(os.path.join(out_dir, f"{name}_params_sample.npy"), flat[idx.to(flat.device)].cpu().numpy())


def run_dprb(args, workload):
    from dpr_scale_b200 import _lib, ops
    from dpr_scale_b200.task.dpr_task import DenseRetrieverTask, _ScoreCE
    from dpr_scale_b200.trainer import Trainer
    from dpr_scale_b200.utils.phase_timer import PhaseTimer

    cfg, B, n, S = WORKLOADS[workload]
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        from dpr_scale_b200.utils.dist_init import init_process_group
        init_process_group(dev)          # NCCL, high-priority stream (see utils/dist_init.py)
    check = None
    if world > 1 and not args.no_selfcheck:
        check = selfcheck(world, rank, dev)
        if rank == 0 and not check.get("ok", True):
            print(f"[bench] MULTI-GPU SELF-CHECK FAILED: {check}", file=sys.stderr)
    task = DenseRetrieverTask(
        transform={}, datamodule=None, shared_model=False, in_batch_negatives=True, warmup_steps=10,
        fp16_grads=(args.grad_dtype == "bf16"),
        model={"_target_": "dpr_scale_b200.models.hf_model.HFEncoder.from_config", "config": cfg,
               "dropout": args.dropout},
        optim={"_target_": "dpr_scale_b200.optim.FusedAdamW", "lr": 1e-5, "betas": [0.9, 0.999], "eps": 1e-8,
               "weight_decay": 0.0})
    trainer = Trainer(max_steps=10 ** 6, gradient_clip_val=2.0, device=dev)
    with contextlib.redirect_stdout(sys.stderr):      # stdout carries exactly ONE line: the JSON result
        trainer.attach(task, None, "fit")
    task.train()
    # fixed dropout streams (the default base mixes in the module's address): with the same arguments every run draws
    # the same masks, so two builds can be compared output for output
    task.query_encoder._drop_base, task.context_encoder._drop_base = 0x5EED0001, 0x5EED0002
    task.context_encoder.activation_chunk = ACT_CHUNK.get(workload, 0) if args.act_chunk < 0 else args.act_chunk
    lean = (workload in LEAN and task.context_encoder.activation_chunk == 0) or args.lean
    task.context_encoder.lean_activations = task.query_encoder.lean_activations = lean
    host_batch = synth_batch(rank, cfg, B, n, S)
    dev_batch = to_device(host_batch, dev)
    lib = _lib.load()

    def sync_all():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def timed(fn, steps, finish=None):
        sync_all()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(steps):
            fn(i)
        if finish is not None:
            finish()                     # still inside the timed region
        e1.record()
        sync_all()
        ms = torch.tensor([e0.elapsed_time(e1)], device=dev)
        if world > 1:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return float(ms) / steps

    # ---- kernel-path number: inputs resident in HBM
    for i in range(args.warmup):
        trainer.training_step(dev_batch, i)
    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    launches0 = ops.launch_count()
    last = {}

    def kernel_step(i):
        # detached: the returned loss holds the step's autograd graph, whose nodes reference both encoders and their
        # activation workspaces; keeping it would keep all of that alive into the stock leg below
        last["loss"] = trainer.training_step(dev_batch, i).detach()

    ms_step = timed(kernel_step, args.steps)
    launches = ops.launch_count() - launches0        # counted inside the C launchers (dprb_launch_count)
    clocks = sampler.stop() if rank == 0 else None
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, last["loss"], task)
    del last

    # ---- roofline leg: the same step, timed again with CUDA events around EVERY GEMM launch.  The query encoder is
    # kept on the main stream here (no two-stream overlap), otherwise launch intervals of the two streams interleave
    # and the per-launch durations would count each other's kernels.
    prof_steps = min(args.steps, 5)
    os.environ["DPRB_NO_STREAM_OVERLAP"] = "1"
    trainer.training_step(dev_batch, 0)
    _lib.check(lib.dprb_gemm_profile_enable(1, 1500 * prof_steps + 64), "profile_enable")
    ms_prof = timed(lambda i: trainer.training_step(dev_batch, i), prof_steps)
    tms, tfl, nl = ctypes.c_double(), ctypes.c_double(), ctypes.c_int64()
    _lib.check(lib.dprb_gemm_profile_read(ctypes.byref(tms), ctypes.byref(tfl), ctypes.byref(nl)), "profile_read")
    _lib.check(lib.dprb_gemm_profile_enable(0, 0), "profile_disable")
    del os.environ["DPRB_NO_STREAM_OVERLAP"]

    # ---- per-phase leg: CUDA events at the phase boundaries of the step (main stream), rank 0's view
    pt = PhaseTimer()
    task.phase_timer = _ScoreCE.phase = pt
    timed(lambda i: trainer.training_step(dev_batch, i), prof_steps)
    phases = pt.summary()
    task.phase_timer = _ScoreCE.phase = None

    # ---- end-to-end number: host (pinned) inputs -> H2D each step, loss read back each step
    # Every step's loss is copied to pinned host memory inside the step and READ one step later (the usual logging lag:
    # the host enqueues step i+1 while the GPU finishes step i); the last one is read before the timer stops.
    losses = []
    loss_host = torch.empty(args.steps + 1, dtype=torch.float32).pin_memory()
    loss_ready = [torch.cuda.Event() for _ in range(args.steps + 1)]

    def read_loss(i):
        loss_ready[i].synchronize()
        losses.append(float(loss_host[i]))

    def e2e_step(i, lag=True):
        b = to_device(host_batch, dev)
        loss = trainer.training_step(b, i)
        loss_host[i:i + 1].copy_(loss.detach().reshape(1), non_blocking=True)   # D2H of the step's loss
        loss_ready[i].record()
        if lag and i > 0:
            read_loss(i - 1)

    e2e_step(args.steps, lag=False)      # one untimed step through the same path (uses the spare slot)
    read_loss(args.steps)
    losses.clear()
    ms_e2e = timed(e2e_step, args.steps, finish=lambda: read_loss(args.steps - 1))

    # ---- N > 1: the same step with the bf16-compressed gradient all-reduce (`fp16_grads`, dpr_task.py:90-92)
    alt = None
    if world > 1:
        other = args.grad_dtype != "bf16"
        trainer.set_grad_compression(other)
        trainer.training_step(dev_batch, 0)
        ms_alt = timed(lambda i: trainer.training_step(dev_batch, i), args.steps)
        trainer.set_grad_compression(not other)
        alt = {"value": B * world / (ms_alt / 1e3), "unit": "pairs/s", "ms_per_step": ms_alt,
               "grad_allreduce": "bf16" if other else "fp32"}

    # ---- end-to-end number INCLUDING the dataloader (single GPU; JSONL -> tokeniser -> pinned -> H2D -> step)
    dl = None
    if world == 1 and not args.no_dataloader:
        try:
            ms_dl = dataloader_leg(trainer, dev, B, n, S, args.steps, args.warmup)
            dl = {"value": B / (ms_dl / 1e3), "unit": "pairs/s", "ms_per_step": ms_dl,
                  "what": "synthetic DPR-format JSONL -> dpr_scale_b200.datamodule (background assembly, Rust tokeniser, "
                          "pinned + side-stream H2D) -> training_step, loss copied to pinned memory every step and read one step later",
                  "host_threads": usable_cores()}
        except Exception as e:  # noqa: the headline numbers above must survive a data-side failure
            dl = {"error": repr(e)[:300]}

    peak_mem = torch.cuda.max_memory_allocated(dev) / 2 ** 30
    if rank != 0:
        if world > 1:
            dist.destroy_process_group()
        return

    # ---- stock HF + PyTorch on the SAME GPU, right after our arm (the 1.5x denominator), its own clock samples
    stock = None
    if world == 1 and not args.no_stock:
        import gc
        del trainer, task, dev_batch
        gc.collect()
        torch.cuda.empty_cache()
        stock = {}
        for dt in ("bf16", "fp16"):
            try:
                stock[dt] = time_stock(cfg, B, n, S, args.dropout, dt, min(args.steps, 10), 3, dev)
            except Exception as e:  # noqa
                stock[dt] = {"error": repr(e)[:300]}

    pairs_step = B * world
    value = pairs_step / (ms_step / 1e3)
    peak_tf, peak_hbm, peak_src = peaks()
    gemm_tflops = (tfl.value / 1e12) / (tms.value / 1e3) if tms.value > 0 else 0.0
    tokens = B * (2 + n) * S
    step_flops = tokens * flops_per_token_train(cfg, S)
    line = {
        "metric": "query+ctx pairs/sec (BERT-base, seq128)" if cfg is BERT_BASE else f"query+ctx pairs/sec ({workload})",
        "value": value, "unit": "pairs/s", "n_gpus": world,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms_step, "higher_is_better": True,
        "scaling": "weak", "vs_baseline": None, "dtype": "bf16", "data": "synthetic",
        "config": {"workload": workload, "model": ("BERT-base" if cfg is BERT_BASE else "RoBERTa-large") + " x2 (query+context, shared_model=false)",
                   "activation_chunk": ACT_CHUNK.get(workload, 0) if args.act_chunk < 0 else args.act_chunk,
                   "lean_activations": bool(lean),
                   "queries_per_gpu": B, "hard_negatives": n, "contexts_per_gpu": B * (1 + n), "seq_len": S,
                   "global_batch": pairs_step, "parallelism": f"dp{world}", "negatives": "global in-batch" if world > 1 else "in-batch",
                   "optimizer": "fused AdamW + clip 2.0 + LambdaLR", "dropout": args.dropout,
                   "grad_allreduce": (args.grad_dtype + (" (reference default: fp16_grads=false)" if args.grad_dtype == "fp32" else " (fp16_grads=true)")) if world > 1 else None,
                   "l2": "working set (tens of GB of activations + 0.9 GB weights/step) exceeds the 50 MB L2; no flush needed"},
        "e2e": {"value": pairs_step / (ms_e2e / 1e3), "unit": "pairs/s", "ms_per_step": ms_e2e,
                "h2d_bytes_per_step": batch_bytes(host_batch), "d2h_bytes_per_step": 4,
                "d2h": "every step's loss copied to pinned host memory in the step, read by the host one step later"},
        "e2e_dataloader": dl,
        "gpu_launches": launches,
        "gpu_launches_how": "dprb_launch_count(): incremented at every kernel launch inside libdprb.so, difference over the timed region",
        "clocks": clocks,
        "peak_mem_gb": peak_mem,
        "roofline": {"bound": "tensor", "kernel": "gemm_bf16_kernel<*,*,*> (wgmma m64n128k16, 128x128 tiles)",
                     "achieved": gemm_tflops, "peak": peak_tf, "unit": "TFLOP/s", "frac": gemm_tflops / peak_tf,
                     "peak_source": peak_src,
                     "traffic": None,
                     "gemm_launches": nl.value,
                     "gemm_ms_per_step": tms.value / prof_steps, "roofline_region_ms_per_step": ms_prof,
                     "gemm_share_of_step": (tms.value / prof_steps) / ms_prof,
                     "step_model_tflops": step_flops / (ms_step / 1e3) / 1e12,
                     "step_frac_of_peak": step_flops / (ms_step / 1e3) / 1e12 / peak_tf},
        "phases": {"ms_per_step": phases, "how": "CUDA events on the main stream at phase boundaries, rank 0, "
                                                 f"{prof_steps} steps; encoders_fwd includes the side-stream query encoder join"},
        "loss_first_last": [losses[0], losses[-1]] if losses else None,
    }
    if check is not None:
        line["selfcheck"] = check
    if alt is not None:
        line["grad_allreduce_" + alt["grad_allreduce"]] = alt
    if stock is not None:
        line["stock_gpu"] = stock
        ok = [v["value"] for v in stock.values() if "value" in v]
        if ok:
            # against the FASTER of the two stock precisions (the conservative ratio)
            line["vs_stock"] = {"ratio": value / max(ok), "e2e_ratio": line["e2e"]["value"] / max(ok),
                                "stock_pairs_per_s": max(ok), "target": 1.5}
    if world == 1 and not args.no_cpu_baseline:
        threads = usable_cores()
        v, sp, kind = time_cpu_reference(cfg, 1, n, S, 2, 1, threads)
        line["cpu_baseline"] = {"value": v, "unit": "pairs/s", "cores": threads, "kind": kind,
                                "sample": f"1 pair/step x 2 steps (+1 warm-up) of {workload}: reference encoder class x2 fp32 "
                                          f"fwd+bwd+clip+AdamW on {threads} host threads"}
    print(json.dumps(line))
    if world > 1:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="dprb", choices=["dprb", "reference", "stock"])
    ap.add_argument("--workload", default="bert-base_s128_b128_n7", choices=sorted(WORKLOADS))
    ap.add_argument("--ref-pairs", type=int, default=1, help="pairs per step of the bounded CPU sample (--impl reference)")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-dataloader", action="store_true", help="skip the end-to-end leg that includes the input pipeline")
    ap.add_argument("--dropout", type=float, default=0.1,
                    help="hidden + attention dropout of both encoders (reference default 0.1, conf/task/model/hf_model.yaml:5)")
    ap.add_argument("--stock-dtype", default="bf16", choices=["bf16", "fp16"])
    ap.add_argument("--no-stock", action="store_true", help="skip the stock HF + PyTorch leg of the default line")
    ap.add_argument("--no-selfcheck", action="store_true", help="skip the NCCL parity self-check at N > 1")
    ap.add_argument("--grad-dtype", default="fp32", choices=["fp32", "bf16"],
                    help="gradient all-reduce precision at N > 1 (fp32 = the reference default fp16_grads=false)")
    ap.add_argument("--lean", action="store_true", help="lean activations (save_for_backward = 2) whatever the workload")
    ap.add_argument("--act-chunk", type=int, default=-1, help="override the activation chunk (sequences) of the context encoder")
    ap.add_argument("--dump-outputs", default=None, metavar="DIR",
                    help="after the timed steps, write what the last timed step computed to DIR/<name>.npy")
    args = ap.parse_args()
    if args.impl == "reference":
        return run_reference(args, args.workload)
    if args.impl == "stock":
        return run_stock(args, args.workload)
    return run_dprb(args, args.workload)


if __name__ == "__main__":
    main()
