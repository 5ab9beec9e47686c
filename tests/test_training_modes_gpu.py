"""The encoder's training modes with dropout on, against float64.

Backward has to replay exactly what forward did: the same dropout masks at every site, under the seed of the forward it
belongs to.  Every check here runs in train mode at p = 0.1 on tiny BERT and RoBERTa models of 5 layers (buckets of 1
and 3 layers leave uneven ranges), with non-zero biases and LayerNorm parameters, ragged padding and S in {64, 200}:

  * lean activations (save_for_backward = 2: backward re-runs each attention forward and rebuilds GELU from the saved
    pre-activation) against the float64 oracle fed the masks of `last_dropout`, and against full mode under one seed;
  * RoBERTa-large (H 1024, 16 heads, 24 layers) in lean mode with dropout at S = 256, the benchmark's workload;
  * activation chunking: forward per chunk without saving, backward re-runs each chunk under that chunk's seed;
  * the shared encoder (shared_model=True): two live forwards with their own seeds back-propagate into one arena;
  * the layer-bucketed backward (`bwd_chunk_layers` + `grad_sync`) that feeds the multi-GPU gradient all-reduce, on one
    GPU with a recorder as `grad_sync`: the slices tile the arena once, top layer first; the hook fires only during the
    last outstanding backward; nothing writes into a slice after it is handed over;
  * the master -> bf16 shadow cast and the fused optimizers' shadow store, bit for bit against round-to-nearest-even.

Gates: pooled output rel-L2 <= 1e-2 against float64; every parameter gradient cosine >= 0.999 and rel-L2 <= 3e-2
(tests/test_long_seq_gpu._check_grads); RoBERTa-large with tests/test_realdims_gpu.py's probe gates; schedules that
only reorder fp32 atomics (chunking, buckets) within 1e-5 rel-L2; outputs bitwise where the arithmetic is identical.
"""
import time

import numpy as np
import pytest
import torch

from tests import realdims
from tests.test_dropout_gpu import P, _masks
from tests.test_long_seq_gpu import _check_grads
from tests.util import cosine, rel_l2

pytestmark = pytest.mark.gpu

L, H, HEADS = 5, 128, 2
TINY = dict(vocab_size=64, hidden_size=H, num_hidden_layers=L, num_attention_heads=HEADS, intermediate_size=256)
KINDS = {
    "bert": (dict(TINY, model_type="bert", max_position_embeddings=256),
             {"layers": L, "heads": HEADS, "ln_eps": 1e-12, "pad_id": 0, "roberta": False}),
    "roberta": (dict(TINY, model_type="roberta", max_position_embeddings=258, type_vocab_size=1, pad_token_id=1,
                     layer_norm_eps=1e-5),
                {"layers": L, "heads": HEADS, "ln_eps": 1e-5, "pad_id": 1, "roberta": True}),
}
# lean vs full mode under one seed, per tensor: the two differ only in the bf16 rounding of the saved FFN
# pre-activation from which lean backward rebuilds gelu / gelu' (globally 2.8e-3 .. 3.1e-3).  The query weight and bias
# gradients are sums of dQ over tokens whose terms largely cancel, so that rounding shows there first: measured worst
# 6.0e-3 (query bias), against at most 4.6e-3 for every other tensor (layer 0's key weight, layer 1's FFN input bias).
LEAN_VS_FULL, LEAN_VS_FULL_QUERY = 5e-3, 1.5e-2
SEEDS = (0x5EED0001, 0xDEADBEEF12345, 2 ** 63 + 7)   # forced dropout seeds of one step's forwards


def _perturb(module, seed, scale=0.02):
    with torch.no_grad():                 # non-zero biases / LayerNorm parameters
        gen = torch.Generator().manual_seed(seed)
        for p in module.parameters():
            p.add_(scale * torch.randn(p.shape, generator=gen))


def _model(kind, lean=False):
    from dpr_scale_b200.models.hf_model import HFEncoder
    cfg, ocfg = KINDS[kind]
    enc = HFEncoder.from_config(cfg, dropout=P, seed=3)
    _perturb(enc, 4)
    sd = {k: v.detach().clone() for k, v in enc.state_dict().items()}
    enc = enc.cuda().train()
    enc.lean_activations = lean
    return enc, sd, ocfg


def _tokens(kind, N, S, seed):
    pad = KINDS[kind][0].get("pad_token_id", 0)
    gen = torch.Generator().manual_seed(seed)
    lens = torch.randint(S // 4, S + 1, (N,), generator=gen)
    lens[0] = S                           # the last position is used
    ids = torch.randint(3, 64, (N, S), generator=gen)
    am = (torch.arange(S).unsqueeze(0) < lens.unsqueeze(1)).long()
    tok = {"input_ids": ids * am + pad * (1 - am), "attention_mask": am}
    if kind == "bert":
        tok["token_type_ids"] = torch.zeros_like(ids)
    return tok


def _probe(N, seed, width=H):
    return torch.randn(N, width, generator=torch.Generator().manual_seed(seed))


def _cat_masks(parts):
    """Per-pass mask dicts of consecutive sequence ranges -> one dict over all of them (concatenated along N)."""
    out = {"emb": torch.cat([m["emb"] for m in parts])}
    for l in (k for k in parts[0] if k != "emb"):
        out[l] = {site: torch.cat([m[l][site] for m in parts]) for site in parts[0][l]}
    return out


def _f64(masks):
    if masks is None:
        return None
    return {k: (v.double() if torch.is_tensor(v) else {s: t.double() for s, t in v.items()}) for k, v in masks.items()}


def _oracle(sd, ocfg, passes):
    """Float64 oracle of sum_i <encode(tokens_i, masks_i), probe_i> over passes through ONE copy of the weights.
    Returns the pooled outputs and the weights, whose .grad hold the reference gradients."""
    from oracle import encoder as oenc
    ref_sd = {k: v.double().clone().requires_grad_(True) for k, v in sd.items()}
    loss, outs = 0.0, []
    for tok, masks, probe in passes:
        r = oenc.encode(ref_sd, ocfg, tok, dropout=_f64(masks))
        loss = loss + (r * probe.double()).sum()
        outs.append(r.detach())
    loss.backward()
    return outs, ref_sd


def _no_dropout_output(sd, ocfg, tok):
    from oracle import encoder as oenc
    return oenc.encode({k: v.double() for k, v in sd.items()}, ocfg, tok)


class _Trace:
    """Wraps one encoder's _run_forward / _run_backward.  Records every forward as (save, p, seed) and counts backward
    calls; `force(*seeds)` hands the next forwards that do not name a seed themselves these seeds, in order."""

    def __init__(self, enc):
        self.fwd, self.bwd, self.forced = [], 0, []
        run_fwd, run_bwd = enc._run_forward, enc._run_backward

        def fwd(tokens, save, train_dropout=None, force_seed=None):
            if force_seed is None and self.forced:
                force_seed = self.forced.pop(0)
            out = run_fwd(tokens, save, train_dropout=train_dropout, force_seed=force_seed)
            self.fwd.append((bool(save),) + tuple(enc.last_dropout))
            return out

        def bwd(*args, **kw):
            self.bwd += 1
            return run_bwd(*args, **kw)

        enc._run_forward, enc._run_backward = fwd, bwd

    def force(self, *seeds):
        self.fwd, self.bwd, self.forced = [], 0, list(seeds)


def _report(tag, **ratios):
    print(tag, "  ".join(f"{k} {v:.3g}" for k, v in ratios.items()))


# ------------------------------------------------------------------ 1. lean activations with dropout
@pytest.mark.parametrize("kind,S", [("bert", 64), ("bert", 200), ("roberta", 64), ("roberta", 200)])
def test_lean_dropout_matches_float64_oracle(kind, S):
    enc, sd, ocfg = _model(kind, lean=True)
    N = 4
    tok, probe = _tokens(kind, N, S, 10 + S), _probe(N, 11)
    enc.zero_grad()
    rep = enc(tok)
    (rep * probe.cuda()).sum().backward()
    torch.cuda.synchronize()
    masks = _masks(*enc.last_dropout, N, S, H, HEADS, L)
    (ref,), ref_sd = _oracle(sd, ocfg, [(tok, masks, probe)])
    err = rel_l2(rep.detach().cpu(), ref)
    off = rel_l2(rep.detach().cpu(), _no_dropout_output(sd, ocfg, tok))
    worst_cs, worst_rel = _check_grads(enc, ref_sd)
    _report(f"lean+dropout {kind} S={S}:", pooled_rel=err, pooled_gate=1e-2, no_dropout_rel=off,
            worst_cos=worst_cs, worst_grad_rel=worst_rel, grad_rel_gate=3e-2)
    assert err <= 1e-2, err
    assert off > 5e-2, off                # the masks really were applied


@pytest.mark.parametrize("kind,S", [("bert", 200), ("roberta", 64)])
def test_lean_and_full_mode_agree_per_tensor(kind, S):
    enc, _, _ = _model(kind)
    trace = _Trace(enc)
    N = 4
    tok, probe = _tokens(kind, N, S, 20 + S), _probe(N, 21).cuda()
    runs = []
    for lean in (False, True):
        enc.lean_activations = lean
        trace.force(SEEDS[0])
        enc.zero_grad()
        rep = enc(tok)
        (rep * probe).sum().backward()
        torch.cuda.synchronize()
        runs.append((rep.detach().clone(), enc.grads.clone()))
        assert trace.fwd == [(True, pytest.approx(P), SEEDS[0])]
    assert torch.equal(runs[0][0], runs[1][0])
    full, lean = runs[0][1], runs[1][1]
    layout = enc.transformer.layout
    views = {name: (full[off:off + int(np.prod(shape))], lean[off:off + int(np.prod(shape))])
             for name, shape, off in layout.entries}
    top = max(float(f.norm()) for f, _ in views.values())
    worst, worst_q, checked = (0.0, ""), (0.0, ""), 0
    for name, (f, g) in views.items():
        if float(f.norm()) < 1e-5 * top:  # analytically zero (key bias): nothing to compare
            continue
        if ".self.query." in name:
            worst_q = max(worst_q, (rel_l2(g, f), name))
        else:
            worst = max(worst, (rel_l2(g, f), name))
        checked += 1
    _report(f"lean vs full {kind} S={S}:", worst_tensor_rel=worst[0], gate=LEAN_VS_FULL, worst_query_rel=worst_q[0],
            query_gate=LEAN_VS_FULL_QUERY, global_rel=rel_l2(lean, full))
    print(f"  worst of {checked} tensors: {worst[1]}, {worst_q[1]}")
    assert checked >= 20
    assert worst[0] <= LEAN_VS_FULL and worst_q[0] <= LEAN_VS_FULL_QUERY, (worst, worst_q)


# ------------------------------------------------------------------ 2. RoBERTa-large, lean + dropout, S = 256
def test_roberta_large_s256_lean_dropout_matches_float64_oracle():
    """The benchmark's lean workload at 3 sequences.  At this random init attention is close to uniform over 256 keys,
    so an attention re-forward under the wrong mask moves the gradients by less than these gates: the tiny models above
    are the check on the mask replay, this one on the 24-layer, 16-head assembly of lean mode with dropout."""
    from dpr_scale_b200.models.hf_model import HFEncoder
    cfg = realdims.ROBERTA_LARGE
    Lr, Hr, Ar = cfg["num_hidden_layers"], cfg["hidden_size"], cfg["num_attention_heads"]
    ocfg = {"layers": Lr, "heads": Ar, "ln_eps": cfg["layer_norm_eps"], "pad_id": cfg["pad_token_id"], "roberta": True}
    enc = HFEncoder.from_config(dict(cfg, model_type="roberta"), dropout=P, seed=5)
    _perturb(enc, 6, scale=0.01)          # HF's init + 0.01 N(0, 1): tests/realdims.py's context-encoder recipe
    sd = {k: v.detach().clone() for k, v in enc.state_dict().items()}
    enc = enc.cuda().train()
    enc.lean_activations = True
    N, S = 3, 256
    tok = realdims.tokens(torch.Generator().manual_seed(7), N, S, cfg["pad_token_id"], "roberta")
    probe = _probe(N, 8, Hr)
    enc.zero_grad()
    rep = enc(tok)
    (rep * probe.cuda()).sum().backward()
    torch.cuda.synchronize()
    rep = rep.detach().cpu()
    masks = _masks(*enc.last_dropout, N, S, Hr, Ar, Lr)
    t0 = time.perf_counter()
    (ref,), ref_sd = _oracle(sd, ocfg, [(tok, masks, probe)])
    t_oracle = time.perf_counter() - t0
    del masks
    enc.eval()
    with torch.no_grad():
        rep0 = enc(tok).cpu()
        ref0 = _no_dropout_output(sd, ocfg, tok)
    err, err0, off = rel_l2(rep, ref), rel_l2(rep0, ref0), rel_l2(rep, ref0)
    top = max(float(v.grad.norm()) for v in ref_sd.values() if v.grad is not None)
    worst, worst_q, bad, checked = (1.0, 0.0, ""), (1.0, 0.0, ""), [], 0
    for k, p in enc.named_parameters():
        r = ref_sd[k].grad
        if r is None or float(r.norm()) < 1e-5 * top:
            continue
        got = p.grad.detach().float().cpu()
        cs, rl = cosine(got, r), rel_l2(got, r)
        checked += 1
        if k.endswith("self.query.bias") or k.endswith("self.query.weight"):
            # cancelling sums of dQ over tokens: tests/test_realdims_gpu.py::_check_probe's looser gate
            worst_q = min(worst_q, (cs, rl, k))
            bad += [] if cs >= 0.995 and rl <= 0.1 else [(k, cs, rl)]
        else:
            worst = min(worst, (cs, rl, k))
            bad += [] if cs >= 0.999 and rl <= 4e-2 else [(k, cs, rl)]
    print(f"roberta-large lean+dropout S={S}: pooled rel {err:.3g} (gate 1e-2; without dropout {err0:.3g}, "
          f"against the no-dropout oracle {off:.3g}), {checked} tensors, worst {worst} (gates 0.999 / 4e-2), "
          f"worst query {worst_q} (gates 0.995 / 0.1), float64 CPU oracle {t_oracle:.1f} s")
    assert err <= 1e-2 and err0 <= 1e-2, (err, err0)
    assert off > 5e-2, off                # the masks really were applied
    assert not bad, bad
    assert checked >= 15 * Lr


# ------------------------------------------------------------------ 3. activation chunking with dropout
@pytest.mark.parametrize("kind,S,lean", [("bert", 200, False), ("roberta", 64, True)])
def test_activation_chunking_replays_each_chunks_seed(kind, S, lean):
    enc, sd, ocfg = _model(kind, lean=lean)
    trace = _Trace(enc)
    N, chunk = 8, 3                       # chunks of 3, 3, 2
    starts = list(range(0, N, chunk))
    tok, probe = _tokens(kind, N, S, 30 + S), _probe(N, 31)
    enc.activation_chunk = chunk
    enc.zero_grad()
    rep = enc(tok)
    (rep * probe.cuda()).sum().backward()
    torch.cuda.synchronize()
    rep = rep.detach().clone()
    g_chunked = enc.grads.clone()
    fwd = [t for t in trace.fwd if not t[0]]
    rec = [t for t in trace.fwd if t[0]]
    seeds = [s for _, _, s in fwd]
    assert len(fwd) == len(rec) == trace.bwd == len(starts) and len(set(seeds)) == len(starts)
    assert all(p == pytest.approx(P) for _, p, _ in trace.fwd)
    assert [s for _, _, s in rec] == seeds          # backward re-runs every chunk under its own seed

    # against float64, each chunk's masks concatenated along N
    parts = [_masks(P, s, min(chunk, N - lo), S, H, HEADS, L) for s, lo in zip(seeds, starts)]
    (ref,), ref_sd = _oracle(sd, ocfg, [(tok, _cat_masks(parts), probe)])
    err = rel_l2(rep.cpu(), ref)
    worst_cs, worst_rel = _check_grads(enc, ref_sd)

    # against each chunk encoded on its own (unchunked autograd path) under that chunk's seed
    enc.activation_chunk = 0
    trace.force(*seeds)
    enc.zero_grad()
    outs = []
    for lo in starts:
        r = enc({k: v[lo:lo + chunk] for k, v in tok.items()})
        (r * probe[lo:lo + chunk].cuda()).sum().backward()
        outs.append(r.detach())
    torch.cuda.synchronize()
    assert [s for _, _, s in trace.fwd] == seeds
    d_sum = rel_l2(g_chunked, enc.grads)
    _report(f"chunking {kind} S={S} lean={lean}:", pooled_rel=err, pooled_gate=1e-2, worst_cos=worst_cs,
            worst_grad_rel=worst_rel, grad_rel_gate=3e-2, vs_per_chunk_sum=d_sum, sum_gate=1e-5)
    assert err <= 1e-2, err
    assert torch.equal(rep, torch.cat(outs))
    assert d_sum <= 1e-5, d_sum          # fp32 atomic order only


# ------------------------------------------------------------------ 4. shared encoder with dropout
def _shared_task(kind, lean):
    from dpr_scale_b200.task.dpr_task import DenseRetrieverTask
    cfg, ocfg = KINDS[kind]
    task = DenseRetrieverTask(transform={}, datamodule=None, optim={}, shared_model=True, softmax_temperature=1.0,
                              model={"_target_": "dpr_scale_b200.models.hf_model.HFEncoder.from_config",
                                     "config": cfg, "dropout": P})
    task.trainer = None
    task.setup("fit")
    enc = task.query_encoder
    assert enc is task.context_encoder
    _perturb(enc, 12)
    sd = {k: v.detach().clone() for k, v in enc.state_dict().items()}
    task = task.cuda().train()
    enc.lean_activations = lean
    return task, enc, sd, ocfg


@pytest.mark.parametrize("kind,S,lean", [("bert", 64, False), ("roberta", 200, True)])
def test_shared_encoder_dropout_matches_float64_oracle(kind, S, lean):
    task, enc, sd, ocfg = _shared_task(kind, lean)
    trace = _Trace(enc)
    N = 4
    qtok, ctok = _tokens(kind, N, S, 40 + S), _tokens(kind, N, S, 41 + S)
    pq, pc = _probe(N, 42), _probe(N, 43)
    enc.zero_grad()
    q, c = task(qtok, ctok)
    assert enc._ws_pool.leased == 2 and enc._pending_bwd == 2      # both forwards alive until backward
    ((q * pq.cuda()).sum() + (c * pc.cuda()).sum()).backward()
    torch.cuda.synchronize()
    assert enc._ws_pool.leased == 0 and enc._pending_bwd == 0 and trace.bwd == 2
    (_, p_q, s_q), (_, p_c, s_c) = trace.fwd
    assert s_q != s_c
    (rq, rc), ref_sd = _oracle(sd, ocfg, [(qtok, _masks(p_q, s_q, N, S, H, HEADS, L), pq),
                                          (ctok, _masks(p_c, s_c, N, S, H, HEADS, L), pc)])
    eq, ec = rel_l2(q.detach().cpu(), rq), rel_l2(c.detach().cpu(), rc)
    worst_cs, worst_rel = _check_grads(enc, ref_sd)
    _report(f"shared {kind} S={S} lean={lean}:", query_rel=eq, context_rel=ec, pooled_gate=1e-2,
            worst_cos=worst_cs, worst_grad_rel=worst_rel, grad_rel_gate=3e-2)
    assert eq <= 1e-2 and ec <= 1e-2, (eq, ec)


# ------------------------------------------------------------------ 5. layer-bucketed backward on one GPU
BUCKET_CASES = {   # mode: (kind, S, sequences per pass); every mode runs lean with dropout
    "lean": ("bert", 200, 4),
    "chunked": ("roberta", 64, 8),
    "shared": ("roberta", 200, 4),
}


def _bucket_step(enc, trace, mode, k, inputs):
    """One step's forward + backward with buckets of k layers (k = 0: unbucketed).  Returns the final gradient arena,
    the pooled outputs and what the grad_sync recorder saw: (lo, hi, backward call, pending backwards, snapshot)."""
    seen = []

    def grad_sync(e, lo, hi):
        torch.cuda.current_stream().synchronize()
        seen.append((lo, hi, trace.bwd, e._pending_bwd, e.grads[lo:hi].clone()))

    enc.bwd_chunk_layers = k
    enc.grad_sync = grad_sync if k else None
    enc.activation_chunk = 3 if mode == "chunked" else 0
    trace.force(*SEEDS)
    enc.zero_grad()
    outs = [enc(tok) for tok, _ in inputs]
    sum((o * probe.cuda()).sum() for o, (_, probe) in zip(outs, inputs)).backward()
    torch.cuda.synchronize()
    enc.grad_sync = None
    return enc.grads.clone(), [o.detach() for o in outs], seen


@pytest.mark.parametrize("k", [1, 3, L])
@pytest.mark.parametrize("mode", list(BUCKET_CASES))
def test_bucketed_backward_hands_over_finished_slices_once(mode, k):
    kind, S, N = BUCKET_CASES[mode]
    enc, _, _ = _model(kind, lean=True)
    trace = _Trace(enc)
    npass = 2 if mode == "shared" else 1
    inputs = [(_tokens(kind, N, S, 50 + i), _probe(N, 60 + i)) for i in range(npass)]
    g_ref, out_ref, seen = _bucket_step(enc, trace, mode, 0, inputs)
    assert seen == []
    g, out, seen = _bucket_step(enc, trace, mode, k, inputs)
    assert all(torch.equal(a, b) for a, b in zip(out, out_ref))   # same seeds, same forward
    assert all(p == pytest.approx(P) for _, p, _ in trace.fwd)
    lay = enc.transformer.layout
    bounds = [(lo, hi) for lo, hi, *_ in seen]
    # tiles [0, total) exactly once, top layer first, the embeddings (with layer 0) in the last slice
    assert bounds[0][1] == lay.total and bounds[-1][0] == 0, bounds
    assert all(a[0] == b[1] for a, b in zip(bounds, bounds[1:])), bounds
    assert bounds[-1][1] == lay.off_layer0 + lay.layer_stride, bounds
    layers = [(hi - max(lo, lay.off_layer0)) / lay.layer_stride for lo, hi in bounds]
    assert all(n == int(n) and 1 <= n <= k for n in layers), layers
    assert len(bounds) == 1 + -(-(L - 1) // k), bounds
    # only the last outstanding backward hands slices over (shared: the second pass; chunked: the last chunk)
    assert trace.bwd == (3 if mode == "chunked" else npass)
    assert all(call == trace.bwd and pending == 1 for _, _, call, pending, _ in seen), \
        [(call, pending) for _, _, call, pending, _ in seen]
    # nothing writes into a slice after it was handed over
    for lo, hi, _, _, snap in seen:
        assert torch.equal(snap, g[lo:hi]), (lo, hi, float((snap - g[lo:hi]).abs().max()))
    d = rel_l2(g, g_ref)
    _report(f"buckets {mode} k={k}:", slices=len(bounds), vs_unbucketed=d, gate=1e-5)
    assert d <= 1e-5, d                   # split-K atomics only


# ------------------------------------------------------------------ 6. master -> bf16 shadow
def _rne_bf16(bits32):
    """float32 bit patterns (np.uint32) -> bf16 round-to-nearest-even bit patterns (np.uint16), and which are NaN."""
    u = bits32.astype(np.uint64)
    rounded = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)
    nan = ((bits32 & 0x7F800000) == 0x7F800000) & ((bits32 & 0x007FFFFF) != 0)
    return rounded, nan


SPECIALS32 = np.array([
    0x00000000, 0x80000000, 0x7F800000, 0xFF800000,                          # +-0, +-inf
    0x7FC00000, 0xFFC00000, 0x7F800001, 0xFF800001, 0x7FBFFFFF, 0x7FFFFFFF,  # NaNs (low payloads truncate to inf)
    0x00000001, 0x80000001, 0x00007FFF, 0x00008000, 0x00018000, 0x00008001,  # subnormals, ties at the bottom
    0x007FFFFF, 0x807F8000, 0x00400000, 0x00800000, 0x00808000, 0x00818000,  # largest subnormal, FLT_MIN
    0x3F808000, 0x3F818000, 0xBF818000, 0x3F807FFF, 0x3F808001, 0x3F7FFFFF,  # ties to even / odd, carry into exponent
    0x7F7F8000, 0x7F7FFFFF, 0xFF7FFFFF, 0x7F7F7FFF, 0x7F7E8000, 0x4B7FC000,  # overflow to inf, FLT_MAX
], dtype=np.uint32)


def _check_f32_bf16(bits32):
    from dpr_scale_b200 import ops
    x = torch.from_numpy(bits32.view(np.float32).copy()).cuda()
    got = torch.full((x.numel(),), float("nan"), dtype=torch.bfloat16, device="cuda")
    ops.cast_f32_bf16(x, got)
    want = x.to(torch.bfloat16)
    gbits = got.view(torch.int16).cpu().numpy().view(np.uint16)
    wbits = want.view(torch.int16).cpu().numpy().view(np.uint16)
    rne, nan = _rne_bf16(bits32)
    assert (gbits[~nan] == rne[~nan]).all() and (gbits[~nan] == wbits[~nan]).all(), \
        [hex(b) for b in bits32[~nan][gbits[~nan] != rne[~nan]][:8]]
    assert torch.isnan(got[torch.from_numpy(nan).cuda()].float()).all()    # NaN stays NaN, whatever its payload


@pytest.mark.parametrize("n", [0, 1, 2, 3, 4, 5, 6, 7, 1027, (1 << 20) + 3])
def test_cast_f32_bf16_rounds_like_torch(n):
    from dpr_scale_b200 import ops
    rng = np.random.default_rng(n)
    if n == 0:
        src = torch.empty(0, device="cuda")
        dst = torch.full((4,), 3.0, dtype=torch.bfloat16, device="cuda")
        ops.cast_f32_bf16(src, dst)
        assert torch.equal(dst, torch.full_like(dst, 3.0))
        return
    if n < 8:                             # slide every special value through the scalar tail
        for o in range(len(SPECIALS32)):
            _check_f32_bf16(np.resize(np.roll(SPECIALS32, -o), n))
        return
    bits = rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32)
    bits[:n // 2] = (bits[:n // 2] & 0xFFFF0000) | 0x8000                    # half of them exact ties
    bits[-len(SPECIALS32):] = SPECIALS32                                    # and the specials, in the tail too
    bits[:len(SPECIALS32)] = SPECIALS32
    _check_f32_bf16(bits)


@pytest.mark.parametrize("n", [0, 1, 2, 3, 5, 7, 65536, 65536 + 3])
def test_cast_bf16_f32_is_exact(n):
    from dpr_scale_b200 import ops
    if n >= 65536:                        # every bf16 bit pattern, NaN payloads included
        bits = np.arange(n, dtype=np.uint32).astype(np.uint16)
    else:
        bits = np.array([0x7FC1, 0xFF81, 0x0001, 0x8001, 0x7F80, 0xFF80, 0x3F81, 0x007F][:n], dtype=np.uint16)
    src = torch.from_numpy(bits.view(np.int16).copy()).cuda().view(torch.bfloat16)
    dst = torch.full((max(n, 4),), 7.0, device="cuda")
    ops.cast_bf16_f32(src, dst[:n] if n else torch.empty(0, device="cuda"))
    got = dst[:n].view(torch.int32).cpu().numpy().view(np.uint32)
    assert (got == bits.astype(np.uint32) << 16).all()
    assert torch.equal(dst[:n].view(torch.int32), src.to(torch.float32).view(torch.int32))
    assert (dst[n:] == 7.0).all()


@pytest.mark.parametrize("which,n", [("adamw", 100001), ("adamw", 100002), ("madgrad", 100003), ("lamb", 0)])
def test_optimizer_shadow_is_master_rounded_to_nearest_even(which, n):
    """The fused steps write the bf16 shadow the next forward multiplies with; it must be master.to(bf16) exactly
    (HFEncoder.mark_shadow_fresh then skips the recast)."""
    from dpr_scale_b200 import ops
    from tests.test_optim_gpu import SEGMENTS
    if which == "lamb":
        n = sum(SEGMENTS)                 # LAMB arenas are multiples of 4: the plan's chunks cover them
    gen = torch.Generator().manual_seed(n)
    p = (torch.randn(n, generator=gen) * 10 ** torch.empty(n).uniform_(-4, 2, generator=gen)).cuda()
    g = torch.randn(n, generator=gen).cuda()
    s1, s2 = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    shadow = torch.full((n,), float("nan"), dtype=torch.bfloat16, device="cuda")
    if which == "adamw":
        ops.adamw_step(p, g, s1, s2, shadow, 1e-2, 0.9, 0.999, 1e-8, 0.01, 1)
    elif which == "lamb":
        ops.lamb_step(p, g, s1, s2, shadow, ops.LambPlan(SEGMENTS, "cuda"), 1e-2, 0.9, 0.999, 1e-6, 0.01, 10.0,
                      False, False, 1)
    else:
        ops.madgrad_step(p, g, s1, s2, None, shadow, 1e-2, 0.0, 0.01, 1e-6, 0)
    torch.cuda.synchronize()
    bits32 = p.cpu().numpy().view(np.uint32)
    rne, nan = _rne_bf16(bits32)
    assert not nan.any()
    got = shadow.view(torch.int16).cpu().numpy().view(np.uint16)
    bad = np.flatnonzero(got != rne)
    assert bad.size == 0, (bad.size, [(int(i), hex(bits32[i]), hex(got[i]), hex(rne[i])) for i in bad[:4]])
    assert torch.equal(shadow.view(torch.int16), p.to(torch.bfloat16).view(torch.int16))
    # rounding, not truncation, decided a good share of them
    assert ((bits32 >> 16).astype(np.uint16) != rne).mean() > 0.3
