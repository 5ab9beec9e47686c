"""Per-kernel parity checks: CUDA path (through the C ABI) vs the CPU oracle on the same seeded inputs.

Each check returns a dict of error figures and raises AssertionError when a stated tolerance is exceeded.
Used by tests/test_ops_gpu.py (pytest -m gpu) and tools/gpu_diag.py (one subprocess per check).

Tolerances (stated here, per the fp contract of BASELINE.json:north_star):
  * bf16-output kernels: |err| <= 2^-7 * max|ref| + small atol   (one bf16 rounding of the result plus fp32
    accumulation-order noise; inputs are the identical bf16-rounded values on both sides)
  * fp32-output kernels (scoring/CE, optimizer, wgrad): rel <= 1e-4 unless noted.
"""
import math

import torch

from dpr_scale_b200 import ops
from oracle import encoder as oenc
from oracle import task as otask

DEV = "cuda"


def _bf(x):
    return x.to(torch.bfloat16)


def _close(name, got, ref, rtol_max, atol=0.0, out=None):
    got = got.detach().float().cpu()
    ref = ref.detach().float().cpu()
    assert got.shape == ref.shape, f"{name}: shape {got.shape} vs {ref.shape}"
    assert torch.isfinite(got).all(), f"{name}: non-finite values"
    err = float((got - ref).abs().max())
    scale = float(ref.abs().max())
    if out is not None:
        out[name + "_maxerr"] = err
        out[name + "_scale"] = scale
    assert err <= rtol_max * scale + atol, f"{name}: max err {err:.4e} > {rtol_max}*{scale:.4e}+{atol}"
    return err


# ------------------------------------------------------------------ GEMM
def check_gemm(M, N, K, a_mn=False, b_mn=False, epilogue=ops.EPI_BIAS, splits=1, seed=0):
    g = torch.Generator().manual_seed(seed)
    A = _bf(torch.randn(M, K, generator=g))
    B = _bf(torch.randn(N, K, generator=g) * 0.5)
    bias = torch.randn(N, generator=g)
    aux = _bf(torch.randn(M, N, generator=g))
    ref = A.double() @ B.double().T
    res = {}
    Ad = (A.T.contiguous() if a_mn else A).to(DEV)
    Bd = (B.T.contiguous() if b_mn else B).to(DEV)
    lda = M if a_mn else K
    ldb = N if b_mn else K
    bias_d, aux_d = bias.to(DEV), aux.to(DEV)
    if epilogue in (ops.EPI_F32_ATOMIC_ADD, ops.EPI_F32_STORE):
        init = torch.randn(M, N, generator=g)
        out = init.clone().to(DEV)
        use_bias = epilogue == ops.EPI_F32_STORE
        ops.gemm(Ad, Bd, out, M, N, K, lda, ldb, N, a_mn, b_mn, epilogue, bias_d if use_bias else None, splits=splits)
        want = ref + (init.double() if epilogue == ops.EPI_F32_ATOMIC_ADD else bias.double())
        _close("gemm_f32", out, want, 2e-5 * math.sqrt(K), 1e-4, res)
        return res
    out = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
    out2 = torch.empty(M, N, dtype=torch.bfloat16, device=DEV) if epilogue == ops.EPI_BIAS_GELU else None
    use_aux = epilogue in (ops.EPI_BIAS_RESIDUAL, ops.EPI_DGELU)
    use_bias = epilogue != ops.EPI_DGELU
    colsum = torch.ones(N, device=DEV) if epilogue != ops.EPI_BIAS_GELU else None
    ops.gemm(Ad, Bd, out, M, N, K, lda, ldb, N, a_mn, b_mn, epilogue, bias_d if use_bias else None,
             aux_d if use_aux else None, N if use_aux else 0, out2, colsum=colsum)
    torch.cuda.synchronize()
    if epilogue == ops.EPI_BIAS:
        want = ref + bias.double()
    elif epilogue == ops.EPI_BIAS_RESIDUAL:
        want = ref + bias.double() + aux.double()
    elif epilogue == ops.EPI_BIAS_GELU:
        pre = ref + bias.double()
        cdf = 0.5 * (1 + torch.erf(pre / math.sqrt(2)))
        pdf = torch.exp(-0.5 * pre * pre) / math.sqrt(2 * math.pi)
        # out2 = gelu'(pre) (what backward needs); fitted-CDF error <= 1.3e-4 + bf16 rounding
        _close("gemm_dgelu_saved", out2, cdf + pre * pdf, 2 ** -7, 1e-3, res)
        want = oenc.gelu_erf(pre)
    else:  # DGELU: plain multiply by the saved derivative
        want = ref * aux.double()
    _close("gemm_out", out, want, 2 ** -7, 1e-3, res)
    if colsum is not None:  # fused bias-gradient column sums of the (bf16-rounded) output
        _close("gemm_colsum", colsum, 1 + out.double().cpu().sum(0), 1e-5, 1e-3, res)
    return res


def check_gemm_f16_stream(M=384, N=768, K=512, seed=30):
    """The encoder's fp16 residual stream through the GEMM epilogue: bf16 operands, residual aux read as fp16, sum written
    as fp16 (DPRB_GEMM_{AUX,OUT}_F16); and the both-operands-fp16 form of the MMA (a mixed fp16 x bf16 pair is rejected)."""
    g = torch.Generator().manual_seed(seed)
    A = _bf(torch.randn(M, K, generator=g))
    B = _bf(torch.randn(N, K, generator=g) * 0.5)
    bias = torch.randn(N, generator=g)
    aux = (torch.randn(M, N, generator=g) * 3).half()
    res = {}
    out = torch.empty(M, N, dtype=torch.float16, device=DEV)
    ops.gemm(A.to(DEV), B.to(DEV), out, M, N, K, K, K, N, False, False,
             ops.EPI_BIAS_RESIDUAL | ops.GEMM_AUX_F16 | ops.GEMM_OUT_F16, bias.to(DEV), aux.to(DEV), N)
    want = A.double() @ B.double().T + bias.double() + aux.double()
    _close("gemm_f16_stream", out, want, 2 ** -10, 1e-3, res)          # fp16 output: 11 significand bits
    Ah, Bh = A.half(), B.half()
    out2 = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
    ops.gemm(Ah.to(DEV), Bh.to(DEV), out2, M, N, K, K, K, N, False, False, ops.EPI_BIAS | ops.GEMM_A_F16 | ops.GEMM_B_F16,
             bias.to(DEV))
    _close("gemm_f16_ab", out2, Ah.double() @ Bh.double().T + bias.double(), 2 ** -7, 1e-3, res)
    try:
        ops.gemm(Ah.to(DEV), B.to(DEV), out2, M, N, K, K, K, N, False, False, ops.EPI_BIAS | ops.GEMM_A_F16, bias.to(DEV))
        raise AssertionError("mixed fp16 x bf16 operands must be rejected on the host")
    except Exception as e:  # noqa
        assert "fp16 x bf16" in str(e), e
    return res


def check_gemm_lean(M=384, N=512, K=256, seed=40):
    """The lean-activations epilogues: BIAS_GELU | SAVE_PRE (out2 = pre-activation), DGELU_PRE (acc * gelu'(pre) rebuilt
    from the saved pre-activation) and the elementwise gelu_from_pre - against erf-GELU and its exact derivative."""
    g = torch.Generator().manual_seed(seed)
    A = _bf(torch.randn(M, K, generator=g))
    B = _bf(torch.randn(N, K, generator=g) * 0.2)
    bias = torch.randn(N, generator=g)
    res = {}
    out = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
    pre_d = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
    ops.gemm(A.to(DEV), B.to(DEV), out, M, N, K, K, K, N, False, False, ops.EPI_BIAS_GELU | ops.GEMM_SAVE_PRE, bias.to(DEV),
             out2=pre_d)
    pre = A.double() @ B.double().T + bias.double()
    _close("lean_pre", pre_d, pre, 2 ** -7, 1e-3, res)
    _close("lean_act", out, oenc.gelu_erf(pre), 2 ** -7, 1e-3, res)
    _close("lean_gelu_from_pre", ops.gelu_from_pre(pre_d), oenc.gelu_erf(pre_d.double().cpu()), 2 ** -7, 1e-3, res)
    # backward: dH[M, K2] = (dY W) * gelu'(pre) with B read MN-major; pre from the forward call above
    dY = _bf(torch.randn(M, K, generator=g))
    W = _bf(torch.randn(K, N, generator=g) * 0.2)          # [K_in = K, N_out = N] row-major == B(n, k) MN-major
    dH = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
    cs = torch.zeros(N, device=DEV)
    ops.gemm(dY.to(DEV), W.to(DEV), dH, M, N, K, K, N, N, False, True, ops.EPI_DGELU_PRE, None, pre_d, N, colsum=cs)
    x = pre_d.double().cpu()
    cdf = 0.5 * (1 + torch.erf(x / math.sqrt(2)))
    pdf = torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)
    want = (dY.double() @ W.double()) * (cdf + x * pdf)
    _close("lean_dgelu", dH, want, 2 ** -7, 2e-3, res)
    _close("lean_dgelu_colsum", cs, dH.double().cpu().sum(0), 1e-5, 1e-3, res)
    return res


# ------------------------------------------------------------------ LayerNorm / embeddings
def check_ln(T=777, H=768, cls_stride=0, seed=1, f16=False):
    """f16: z arrives in fp16 (written by a DPRB_GEMM_OUT_F16 epilogue) and the fp16 residual copy y_res is requested."""
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(T, H, generator=g) * 2 + 0.3
    z = z.half() if f16 else _bf(z)          # f16: the encoder's residual-stream format (z in / y out in fp16)
    gamma = 1 + 0.1 * torch.randn(H, generator=g)
    beta = 0.1 * torch.randn(H, generator=g)
    eps = 1e-12
    res = {}
    y_res = torch.empty(T, H, dtype=torch.float16, device=DEV) if f16 else None
    y, stats, cls = ops.ln_fwd(z.to(DEV), gamma.to(DEV), beta.to(DEV), eps, cls_stride, y_res)
    zr = z.float().requires_grad_(True)
    gr, br = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    yr = oenc.layer_norm(zr, gr, br, eps)
    _close("ln_y", y, yr, 2 ** -7, 1e-3, res)
    if f16:
        _close("ln_y_res", y_res, yr, 2 ** -10, 1e-3, res)
    if cls_stride:
        _close("ln_cls", cls, yr[::cls_stride], 1e-5, 1e-5, res)
    # backward
    dy = _bf(torch.randn(T, H, generator=g))
    dgamma = torch.zeros(H, device=DEV)
    dbeta = torch.zeros(H, device=DEV)
    dbias = torch.zeros(H, device=DEV)
    if cls_stride:
        ncls = (T + cls_stride - 1) // cls_stride
        dy_cls = torch.randn(ncls, H, generator=g)
        dyr = torch.zeros(T, H)
        dyr[::cls_stride] = dy_cls
        dz = ops.ln_bwd(None, z.to(DEV), stats, gamma.to(DEV), dgamma, dbeta, dbias, dy_cls.to(DEV), cls_stride)
    else:
        dyr = dy.float()
        dz = ops.ln_bwd(dy.to(DEV), z.to(DEV), stats, gamma.to(DEV), dgamma, dbeta, dbias)
    yr.backward(dyr)
    _close("ln_dz", dz, zr.grad, 2 ** -7, 1e-3, res)
    _close("ln_dgamma", dgamma, gr.grad, 1e-4, 1e-3, res)
    _close("ln_dbeta", dbeta, br.grad, 1e-4, 1e-3, res)
    _close("ln_dbias", dbias, dz.float().cpu().sum(0), 1e-4, 1e-3, res)
    if not cls_stride:
        # hidden dropout between the Linear and this LayerNorm: second output dz * mask / (1-p), and the bias gradient
        # is the column sum of THAT (the Linear's own output gradient)
        p_drop, seed0, layer, site = 0.1, 11, 2, 3
        dg2, db2, dbias2 = (torch.zeros(H, device=DEV) for _ in range(3))
        dz2, dzm = ops.ln_bwd(dy.to(DEV), z.to(DEV), stats, gamma.to(DEV), dg2, db2, dbias2, None, 1, p_drop,
                              ops.dropout_site_seed(seed0, layer, site))
        keep = ops.dropout_mask(T, H, p_drop, seed0, layer, site).float()
        scale = 1.0 / (1.0 - round(p_drop * 65536) / 65536.0)
        assert torch.equal(dz2, dz), "ln_bwd: dz must not depend on the dropout site"
        _close("ln_drop_dzm", dzm, dz.float() * keep * scale, 2 ** -7, 1e-3, res)
        _close("ln_drop_dbias", dbias2, dzm.float().cpu().sum(0), 1e-4, 1e-3, res)
        _close("ln_drop_dgamma", dg2, gr.grad, 1e-4, 1e-3, res)
    return res


def check_embed(T=500, H=768, vocab=1000, max_pos=64, type_vocab=2, seed=2, dropout=0.0, y_res=False, roberta_S=0):
    """dropout: embedding dropout (site 0 of layer 0), replayed from dprb_dropout_mask(T, H, p, seed, 0, 0);
    y_res: the fp16 residual-stream copy of the output; type_vocab >= 3 takes the per-element atomic branch of the
    type-table gradient; roberta_S: RoBERTa's pad-derived positions (cumsum of non-pad tokens + pad id) over sequences
    of roberta_S tokens, so the position changes between the rows one warp handles (T above the 4224 warps of the
    grid gives every warp several rows)."""
    g = torch.Generator().manual_seed(seed)
    if roberta_S:
        pad = 1
        max_pos = roberta_S + pad + 1
    word = torch.randn(vocab, H, generator=g) * 0.5
    pos = torch.randn(max_pos, H, generator=g) * 0.5
    typ = torch.randn(type_vocab, H, generator=g) * 0.5
    gamma = 1 + 0.1 * torch.randn(H, generator=g)
    beta = 0.1 * torch.randn(H, generator=g)
    ids = torch.randint(0, vocab, (T,), generator=g)
    ids[:50] = 7  # repeated ids -> atomic accumulation
    tts = torch.randint(0, type_vocab, (T,), generator=g)
    if roberta_S:
        assert T % roberta_S == 0
        ids = torch.randint(2, vocab, (T // roberta_S, roberta_S), generator=g)
        lens = torch.randint(1, roberta_S + 1, (T // roberta_S,), generator=g)
        ids[torch.arange(roberta_S).unsqueeze(0) >= lens.unsqueeze(1)] = pad
        pids = oenc.roberta_position_ids(ids, pad).flatten()
        ids = ids.flatten()
    else:
        pids = torch.arange(T) % max_pos
    eps = 1e-12
    res = {}
    d = lambda t: t.to(DEV)
    dseed = 0xE3B + seed
    yres = torch.empty(T, H, dtype=torch.float16, device=DEV) if y_res else None
    y, stats = ops.embed_ln_fwd(d(ids), d(tts), d(pids), d(word), d(pos), d(typ), d(gamma), d(beta), eps, dropout, dseed,
                                yres)
    wr, pr, tr = (t.clone().requires_grad_(True) for t in (word, pos, typ))
    gr, br = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    yr = oenc.layer_norm((wr[ids] + tr[tts]) + pr[pids], gr, br, eps)
    if dropout:
        keep = ops.dropout_mask(T, H, dropout, dseed, 0, 0).float().cpu()
        yr = yr * keep / (1.0 - round(dropout * 65536) / 65536.0)
    _close("emb_y", y, yr, 2 ** -7, 1e-3, res)
    if y_res:
        _close("emb_y_res", yres, yr, 2 ** -10, 1e-3, res)
    dy = _bf(torch.randn(T, H, generator=g))
    dword, dpos, dtyp = torch.zeros_like(d(word)), torch.zeros_like(d(pos)), torch.zeros_like(d(typ))
    dgamma, dbeta = torch.zeros(H, device=DEV), torch.zeros(H, device=DEV)
    ops.embed_ln_bwd(d(dy), d(ids), d(tts), d(pids), d(word), d(pos), d(typ), d(gamma), stats, dword, dpos, dtyp, dgamma,
                     dbeta, dropout, dseed)
    yr.backward(dy.float())
    _close("emb_dword", dword, wr.grad, 1e-4, 1e-3, res)
    _close("emb_dpos", dpos, pr.grad, 1e-4, 1e-3, res)
    _close("emb_dtype", dtyp, tr.grad, 1e-4, 1e-3, res)
    _close("emb_dgamma", dgamma, gr.grad, 1e-4, 1e-3, res)
    _close("emb_dbeta", dbeta, br.grad, 1e-4, 1e-3, res)
    return res


def check_colsum(T=1000, N=2304, seed=3):
    g = torch.Generator().manual_seed(seed)
    x = _bf(torch.randn(T, N, generator=g))
    out = torch.ones(N, device=DEV)
    ops.colsum(x.to(DEV), out)
    res = {}
    _close("colsum", out, 1 + x.double().sum(0), 1e-5, 1e-3, res)
    return res


# ------------------------------------------------------------------ attention
ATTN_GUARD = 64          # guard rows (ctx, dqkv) / values per head (lse) past the outputs


def _sentinel(shape, dtype=torch.bfloat16):
    """Buffer of all-ones bits (a NaN in bf16 and fp32): an element the kernel does not write stays non-finite."""
    it = torch.int16 if dtype == torch.bfloat16 else torch.int32
    return torch.full(shape, -1, dtype=it, device=DEV).view(dtype)


def _bits(t):
    return t.view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)


def attn_mask(kind, nseq, S, g):
    """int32 [nseq, S] key mask (None for "none"); every sequence keeps at least one valid key.
      random_prefix: a valid prefix of random length in [S/4, S];
      prefix: lengths 1, S - 1, S, and one key into the last 64- and the last 128-key block, in turn;
      holes:  ~70 % random keys and a 20-key interior hole across a 128- (short S: a 64-) key boundary, key 0 kept;
      left:   left padding: the first S/2 keys masked, or (S > 256) exactly the first 128-key block, in turn;
      last:   a single valid key, at position S - 1."""
    if kind == "none":
        return None
    am = torch.ones(nseq, S, dtype=torch.int32)
    if kind == "random_prefix":
        for i in range(nseq):
            am[i, int(torch.randint(max(1, S // 4), S + 1, (1,), generator=g)):] = 0
    elif kind == "prefix":
        lens = [1, max(1, S - 1), S, 64 * ((S - 1) // 64) + 1, 128 * ((S - 1) // 128) + 1]
        for i in range(nseq):
            am[i, lens[i % len(lens)]:] = 0
    elif kind == "holes":
        am = (torch.rand(nseq, S, generator=g) < 0.7).to(torch.int32)
        if S >= 148:
            am[:, 118:138] = 0
        elif S >= 84:
            am[:, 54:74] = 0
        am[:, 0] = 1
    elif kind == "left":
        n0 = [S // 2] + ([128] if S > 256 else [])
        for i in range(nseq):
            am[i, :n0[i % len(n0)]] = 0
    elif kind == "last":
        am[:, :S - 1] = 0
    else:
        raise ValueError(kind)
    return am


def _attn_qkv(nseq, S, heads, qscale, late_max, g):
    """bf16 [nseq*S, 3H] on the device.  qscale multiplies Q: |q.k| / 8 ~ qscale * N(0, 1), up to ~30 at qscale 10.
    late_max: every logit is ~10 * key / S plus noise of ~0.5, so each key block raises every row's running maximum
    (the long forward rescales O and l at every block) and the largest logit of every row sits in the last block."""
    H = heads * 64
    x = torch.randn(nseq * S, 3, heads, 64, device=DEV, generator=g)
    x[:, 0] *= qscale
    if late_max:
        u = torch.full((64,), 0.125, device=DEV)          # unit vector shared by every query and key
        pos = (torch.arange(nseq * S, device=DEV) % S).float() / S
        x[:, 0] = 0.3 * x[:, 0] + 8 * u
        x[:, 1] = 0.3 * x[:, 1] + 10 * pos[:, None, None] * u
    return x.view(nseq * S, 3 * H).to(torch.bfloat16)


def _per_problem(name, got, ref, rtol, atol, out, bound=None):
    """got / ref [n, heads, rows, cols]: max |got - ref| (less `bound`, elementwise) of every (sequence, head) problem
    against rtol * that problem's max|ref| + atol; keeps the worst problem of `name` in out."""
    assert torch.isfinite(got).all(), f"{name}: unwritten or non-finite values"
    err = (got - ref).abs()
    e, sc = err.amax(dim=(-2, -1)).flatten(), ref.abs().amax(dim=(-2, -1)).flatten()
    if bound is not None:   # the worst problem by the plain gate as well, for the record
        out[name + "_plain"] = max(out.get(name + "_plain", 0.0), float((e / (rtol * sc + atol)).max()))
        err = (err - bound).clamp_min(0)
        e = err.amax(dim=(-2, -1)).flatten()
    ratio = e / (rtol * sc + atol)
    i = int(ratio.argmax())
    if float(ratio[i]) >= out.get(name + "_ratio", -1.0):
        out[name + "_ratio"], out[name + "_err"], out[name + "_scale"] = float(ratio[i]), float(e[i]), float(sc[i])


def check_attention(nseq=3, S=128, heads=2, masked=True, seed=4, dropout=0.0, mask=None, qscale=1.0, late_max=False):
    """dprb_attn_fwd / _bwd against a float64 softmax attention of the same bf16 qkv, computed on the device a chunk of
    sequences at a time.  mask: a kind of attn_mask() (default: "random_prefix" if masked, else "none").

    Gates, per (sequence, head) problem against that problem's max|ref|; the worst problem of each is returned as
    <name>_err / _scale / _ratio (err over gate):
      ctx 2^-7 * max + 1e-4 (P is rounded to bf16 before P V, ctx once more);  lse 1e-4 absolute per row;
      dV 2^-6 * max + 1e-5 (P rounded to bf16);  dQ, dK 2^-6 * max + 1e-5 beyond a first-order bound of the error that
      dS = P (dP - D) / 8 inherits from its inputs, elementwise, E_dQ = A |K| and E_dK = A^T |Q| with
      A = P (2^-12 (|dP| + sum_j P |dP|) + dD) / 8: 2^-12 is the relative error of the kernel's P that the lse gate
      allows (1e-4 = 2^-13.3, plus logit rounding), and dD = sum_d |dO| |ctx - ctx_ref| is the error of D =
      rowsum(dO * ctx) that the long backward (S > 256) takes from the bf16 ctx (0 for S <= 256, which rebuilds D from
      P and dP).  Without it dS = 0 rows (one valid key, or a peaked softmax at qscale 10 in the long kernels) would be
      gated on rounding noise alone;
      dbias (fused QKV bias gradient, accumulated into ones) 1e-5 * max|ref| against the column sums of dqkv.
    And exactly: ctx / lse / dqkv start as a NaN sentinel with ATTN_GUARD guard rows (values) past nseq*S: every
    element in range is written and finite, every guard element keeps its bits; dK / dV of masked keys are 0; K / V of
    masked keys times 100 leave ctx and lse unchanged; replacing the qkv, mask and dctx of the odd sequences leaves the
    even sequences' ctx and lse unchanged (an all-ones mask there stands in for no mask); both forwards and the long
    backward are bitwise repeatable.  The S <= 256 backward adds dQ with shared-memory atomics from two warpgroups:
    its repeatability is returned as bwd_repeatable, not gated.

    Not covered: a sequence with no valid key (no tokenizer path produces one).  From the code the forward gives ctx 0
    and lse -inf there and the backward NaN (exp2(-inf - -inf)), which the fused dbias spreads to every column."""
    kind = mask if mask is not None else ("random_prefix" if masked else "none")
    g = torch.Generator().manual_seed(seed)
    gd = torch.Generator(device=DEV).manual_seed(seed)
    H, T, G = heads * 64, nseq * S, ATTN_GUARD
    qkv = _attn_qkv(nseq, S, heads, qscale, late_max, gd)
    am = attn_mask(kind, nseq, S, g)
    amd = am.to(DEV) if am is not None else None
    dctx = torch.randn(T, H, device=DEV, generator=gd).to(torch.bfloat16)
    dseed, site, keep = 0x1234567 + seed, 0, None
    if dropout > 0:  # attention-probability dropout: export the (never stored) mask and replay it in the reference
        site = ops.dropout_site_seed(dseed, 3, 1)
        keep = ops.dropout_mask(nseq * heads * S, S, dropout, dseed, 3, 1).view(nseq, heads, S, S)

    def fwd(x, m):
        cb, lb = _sentinel((T + G, H)), _sentinel((nseq * heads * S + G,), torch.float32)
        ops.attn_fwd(x, m, nseq, S, heads, True, dropout, site, ctx=cb[:T], lse=lb[:T * heads].view(nseq, heads, S))
        return cb, lb

    def bwd(dbias):
        db = _sentinel((T + G, 3 * H))
        ops.attn_bwd(qkv, amd, ctx, lse, dctx, nseq, S, heads, dbias, dropout, site, dqkv=db[:T])
        return db

    ctx_b, lse_b = fwd(qkv, amd)
    ctx, lse = ctx_b[:T], lse_b[:T * heads].view(nseq, heads, S)
    dbias = torch.ones(3 * H, device=DEV)
    dqkv_b = bwd(dbias)
    dqkv = dqkv_b[:T]
    res = {}

    # exact properties
    ctx_b2, lse_b2 = fwd(qkv, amd)
    assert torch.equal(_bits(ctx_b2), _bits(ctx_b)) and torch.equal(_bits(lse_b2), _bits(lse_b)), \
        "attn_fwd is not bitwise repeatable"
    del ctx_b2, lse_b2
    dqkv_b2 = bwd(None)
    res["bwd_repeatable"] = float(torch.equal(_bits(dqkv_b2), _bits(dqkv_b)))
    assert S <= 256 or res["bwd_repeatable"], "the S > 256 attn_bwd is not bitwise repeatable"
    del dqkv_b2
    for name, buf in (("ctx", ctx_b[T:]), ("lse", lse_b[T * heads:]), ("dqkv", dqkv_b[T:])):
        assert bool((_bits(buf) == -1).all()), f"{name}: written past nseq * S"
    assert torch.isfinite(lse).all(), "lse: unwritten or non-finite values"
    if am is not None and bool((am == 0).any()):
        off = (amd == 0).flatten()
        assert float(dqkv[off, H:].float().abs().max()) == 0.0, "dK / dV of masked keys must be exactly zero"
        big = qkv.clone()
        big[off, H:] = (big[off, H:].float() * 100).to(torch.bfloat16)
        cb, lb = fwd(big, amd)
        assert torch.equal(_bits(cb), _bits(ctx_b)) and torch.equal(_bits(lb), _bits(lse_b)), \
            "K / V of masked keys changed ctx or lse"
        del big, cb, lb
    if nseq > 1:
        odd = (torch.arange(T, device=DEV) // S) % 2 == 1
        other = qkv.clone()
        other[odd] = torch.randn(int(odd.sum()), 3 * H, device=DEV, generator=gd).to(torch.bfloat16) * 3
        am2 = amd.clone() if amd is not None else torch.ones(nseq, S, dtype=torch.int32, device=DEV)
        am2[1::2] = attn_mask("holes", nseq, S, g).to(DEV)[1::2]
        cb, lb = fwd(other, am2)
        ev = ~odd
        assert torch.equal(_bits(cb[:T][ev]), _bits(ctx[ev])), "ctx depends on other sequences"
        assert torch.equal(_bits(lb[:T * heads].view(nseq, heads, S)[0::2]), _bits(lse[0::2])), \
            "lse depends on other sequences"
        del other, am2, cb, lb

    # float64 reference, a chunk of sequences at a time (at most 2^23 attention probabilities per chunk)
    step = max(1, (1 << 23) // (heads * S * S))
    for s0 in range(0, nseq, step):
        s1 = min(nseq, s0 + step)
        n, r0, r1 = s1 - s0, s0 * S, s1 * S
        x = qkv[r0:r1].double().view(n, S, 3, heads, 64)
        q, k, v = (x[:, :, i].transpose(1, 2) for i in range(3))          # n, heads, S, 64
        sc = q @ k.transpose(-1, -2) / 8.0
        if amd is not None:
            sc = sc.masked_fill(amd[s0:s1].view(n, 1, 1, S) == 0, float("-inf"))
        if late_max:
            blk = 128 if S > 256 else 64
            assert bool((sc.argmax(-1) >= blk * ((S - 1) // blk)).all()), "late_max: a row peaks before the last block"
        lse_r = torch.logsumexp(sc, -1)
        p = torch.exp(sc - lse_r[..., None])
        mult = None if keep is None else keep[s0:s1].double() / (1.0 - round(dropout * 65536) / 65536.0)
        pm = p if mult is None else p * mult
        o = pm @ v
        dO = dctx[r0:r1].double().view(n, S, heads, 64).transpose(1, 2)
        dp = dO @ v.transpose(-1, -2)
        if mult is not None:
            dp = dp * mult
        ds = p * (dp - (p * dp).sum(-1, keepdim=True)) / 8.0
        got = dqkv[r0:r1].view(n, S, 3, heads, 64)
        c_got = ctx[r0:r1].view(n, S, heads, 64).transpose(1, 2).double()
        dD = (dO.abs() * (c_got - o).abs()).sum(-1, keepdim=True) if S > 256 else 0.0
        A = p * (2 ** -12 * (dp.abs() + (p * dp.abs()).sum(-1, keepdim=True)) + dD) / 8.0
        _per_problem("ctx", c_got, o, 2 ** -7, 1e-4, res)
        _per_problem("lse", lse[s0:s1].double()[..., None], lse_r[..., None], 0.0, 1e-4, res)
        _per_problem("dq", got[:, :, 0].transpose(1, 2).double(), ds @ k, 2 ** -6, 1e-5, res, A @ k.abs())
        _per_problem("dk", got[:, :, 1].transpose(1, 2).double(), ds.transpose(-1, -2) @ q, 2 ** -6, 1e-5, res,
                     A.transpose(-1, -2) @ q.abs())
        _per_problem("dv", got[:, :, 2].transpose(1, 2).double(), pm.transpose(-1, -2) @ dO, 2 ** -6, 1e-5, res)
        del x, q, k, v, sc, p, pm, o, dO, dp, ds, got, c_got, A, mult
    want = 1 + dqkv.double().sum(0)
    res["dbias_err"], res["dbias_scale"] = float((dbias.double() - want).abs().max()), float(want.abs().max())
    res["dbias_ratio"] = res["dbias_err"] / (1e-5 * res["dbias_scale"])
    bad = [f"{k[:-6]}: err {res[k[:-6] + '_err']:.3e} at max|ref| {res[k[:-6] + '_scale']:.3e} ({v:.2f} x gate)"
           for k, v in res.items() if k.endswith("_ratio") and v > 1.0]
    assert not bad, "; ".join(bad)
    return res


# ------------------------------------------------------------------ scoring + CE
def check_score_ce(Q=37, C=250, d=768, inv_t=2.0, q0=8, nq=16, c0=40, nc=100, seed=5, pair=False):
    """Fused scoring + CE on the tensor-core single pass (tiles recomputed in backward, no logits in HBM unless asked;
    d % 8 != 0 zero-padded) against oracle/task.py (dpr_task.py:98-105, :197-212)."""
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(Q, d, generator=g)
    c = torch.randn(C, d, generator=g)
    mask = torch.rand(C, generator=g) < 0.1
    labels = torch.randint(0, C, (Q,), generator=g)
    mask[labels] = False
    res = {}
    d_ = lambda t: t.to(DEV)
    pm = None
    if pair:
        pm = torch.rand(Q, C, generator=g) < 0.2
        pm[torch.arange(Q), labels] = False
    qr, cr = q.clone().requires_grad_(True), c.clone().requires_grad_(True)
    full_mask = mask.unsqueeze(0).expand(Q, -1) if pm is None else (pm | mask.unsqueeze(0))
    logits_r = otask.sim_score(qr, cr, full_mask) * inv_t
    loss_r = torch.nn.functional.cross_entropy(logits_r, labels)
    loss_r.backward()
    fin = torch.isfinite(logits_r)
    pmd = None if pm is None else d_(pm.to(torch.uint8))

    def compare(tag, loss_sum, lse, logits, dq, dc):
        if logits is not None:
            assert torch.equal(torch.isfinite(logits.cpu()), fin)
            _close(tag + "logits", torch.where(fin, logits.cpu(), torch.zeros(())), torch.where(fin, logits_r.detach(), torch.zeros(())), 1e-5, 1e-3, res)
        _close(tag + "lse", lse, torch.logsumexp(logits_r.detach(), 1), 1e-5, 1e-3, res)
        res[tag + "loss_abs_err"] = abs(float(loss_sum) / Q - float(loss_r))
        assert res[tag + "loss_abs_err"] <= 1e-4 * max(1.0, abs(float(loss_r))), res
        _close(tag + "dq", dq, qr.grad[q0:q0 + nq], 1e-4, 1e-6, res)
        _close(tag + "dc", dc, cr.grad[c0:c0 + nc], 1e-4, 1e-6, res)

    # training form: no logits, backward recomputes the local tiles
    loss_sum, lse, logits, ctx = ops.score_fwd(d_(q), d_(c), d_(mask.to(torch.uint8)), d_(labels), inv_t, False, pmd, (nq, nc))
    assert logits is None and ctx is not None
    dq, dc = ops.score_bwd(ctx, 1.0, inv_t, q0, nq, c0, nc)
    compare("tc_", loss_sum, lse, None, dq, dc)
    # evaluation form: logits requested; a second call on the same shapes (counters must have been reset)
    loss_sum2, lse2, logits2, _ = ops.score_fwd(d_(q), d_(c), d_(mask.to(torch.uint8)), d_(labels), inv_t, True, pmd)
    compare("tc2_", loss_sum2, lse2, logits2, dq, dc)
    assert torch.equal(lse2, lse)
    return res


def check_score_ce_no_queries(C=33, d=128):
    """Q = 0: the forward launches nothing and returns a zero loss sum, an empty lse and empty logits."""
    c = torch.randn(C, d, device=DEV)
    q = torch.empty(0, d, device=DEV)
    labels = torch.empty(0, dtype=torch.int64, device=DEV)
    loss_sum, lse, logits, _ = ops.score_fwd(q, c, None, labels, 1.0, True)
    assert float(loss_sum) == 0.0 and lse.shape == (0,) and logits.shape == (0, C)
    return {"loss_sum": float(loss_sum)}


# ------------------------------------------------------------------ optimizer
def check_adamw(n=100003, seed=6):
    g = torch.Generator().manual_seed(seed)
    p = torch.randn(n + 1, generator=g)[:n].clone()
    res = {}
    pd, md, vd = p.to(DEV), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    shadow = torch.empty(n, dtype=torch.bfloat16, device=DEV)
    pr, mr, vr = p.clone(), torch.zeros(n), torch.zeros(n)
    for step in range(1, 4):
        gr = torch.randn(n, generator=g) * 3
        gd = gr.to(DEV)
        ss = torch.zeros(1, device=DEV)
        ops.sumsq(gd, ss)
        ops.adamw_step(pd, gd, md, vd, shadow, 1e-3, 0.9, 0.999, 1e-8, 0.01, step, 0.5, ss, 2.0)
        coef, total = otask.clip_coef([gr * 0.5], 2.0)
        res["norm_rel_err"] = abs(math.sqrt(float(ss)) * 0.5 - total) / total
        assert res["norm_rel_err"] < 1e-4
        otask.adamw_step(pr, gr * 0.5 * coef, mr, vr, step, 1e-3, weight_decay=0.01)
    _close("adam_p", pd, pr, 1e-5, 1e-6, res)
    _close("adam_m", md, mr, 1e-4, 1e-7, res)
    _close("adam_v", vd, vr, 1e-4, 1e-9, res)
    _close("adam_shadow", shadow, pr, 2 ** -8, 1e-6, res)
    return res


CHECKS = {
    "gemm_kk_bias_irregular": lambda: check_gemm(300, 520, 200),
    "gemm_kk_bias_big": lambda: check_gemm(1024, 768, 768),
    "gemm_kk_gelu": lambda: check_gemm(512, 1024, 256, epilogue=ops.EPI_BIAS_GELU),
    "gemm_kk_residual": lambda: check_gemm(384, 768, 512, epilogue=ops.EPI_BIAS_RESIDUAL),
    "gemm_kmn_dgelu": lambda: check_gemm(384, 512, 256, b_mn=True, epilogue=ops.EPI_DGELU),
    "gemm_kmn_bias": lambda: check_gemm(300, 520, 200, b_mn=True),
    "gemm_mnk_bias": lambda: check_gemm(256, 512, 320, a_mn=True),
    "gemm_mnmn_atomic_split": lambda: check_gemm(768, 768, 4096, a_mn=True, b_mn=True, epilogue=ops.EPI_F32_ATOMIC_ADD, splits=0),
    "gemm_mnmn_atomic_irregular": lambda: check_gemm(200, 264, 1000, a_mn=True, b_mn=True, epilogue=ops.EPI_F32_ATOMIC_ADD, splits=3),
    "gemm_kk_f32_store": lambda: check_gemm(130, 260, 96, epilogue=ops.EPI_F32_STORE),
    "gemm_many_tiles": lambda: check_gemm(4096, 2304, 768),
    "ln_768": lambda: check_ln(777, 768),
    "ln_1024_cls": lambda: check_ln(512, 1024, cls_stride=64),
    "ln_128": lambda: check_ln(100, 128),
    "ln_768_f16": lambda: check_ln(777, 768, f16=True),
    "ln_1024_cls_f16": lambda: check_ln(512, 1024, cls_stride=64, f16=True),
    "gemm_lean_epilogues": lambda: check_gemm_lean(),
    "gemm_lean_epilogues_big": lambda: check_gemm_lean(1024, 3072, 768, seed=41),
    "gemm_f16_stream": lambda: check_gemm_f16_stream(),
    "gemm_f16_stream_big": lambda: check_gemm_f16_stream(1024, 768, 3072, seed=31),
    "embed": lambda: check_embed(),
    "colsum": lambda: check_colsum(),
    "attn_128_masked": lambda: check_attention(3, 128, 2, True),
    "attn_64_nomask": lambda: check_attention(2, 64, 3, False),
    "attn_100_masked": lambda: check_attention(2, 100, 2, True),
    "attn_256_masked": lambda: check_attention(2, 256, 1, True),
    "score_ce": lambda: check_score_ce(),
    "score_ce_small": lambda: check_score_ce(Q=8, C=16, d=128, inv_t=1.0, q0=0, nq=8, c0=0, nc=16),
    "adamw": lambda: check_adamw(),
}

# attention (S <= 128) extra shapes: many problems, heads=12
CHECKS["score_ce_8gpu_shape"] = lambda: check_score_ce(Q=1024, C=8192, d=768, inv_t=0.125, q0=256, nq=128, c0=2048,
                                                       nc=1024, seed=16)     # cfg 3: global 1024 x 8192 scores per rank
CHECKS["score_ce_pair_mask"] = lambda: check_score_ce(Q=130, C=300, d=128, inv_t=1.0, q0=1, nq=129, c0=0, nc=300, seed=17, pair=True)
CHECKS["score_ce_cfg4_shape"] = lambda: check_score_ce(Q=512, C=1024, d=1024, inv_t=1.0, q0=64, nq=64, c0=0, nc=1024, seed=18)
CHECKS["score_ce_odd_d"] = lambda: check_score_ce(Q=9, C=33, d=100, inv_t=1.0, q0=0, nq=9, c0=0, nc=33, seed=19)   # d % 8 != 0 -> zero-padded to 104
CHECKS["score_ce_no_queries"] = lambda: check_score_ce_no_queries()
CHECKS["score_ce_ragged_splits"] = lambda: check_score_ce(Q=70, C=1999, d=200, inv_t=0.5, q0=3, nq=60, c0=17, nc=1500,
                                                          seed=17)
CHECKS["attn_tc_many"] = lambda: check_attention(40, 128, 12, True, seed=9)
CHECKS["attn_tc_s64_many"] = lambda: check_attention(33, 64, 4, True, seed=10)
CHECKS["attn_tc_s37"] = lambda: check_attention(5, 37, 2, True, seed=11)
CHECKS["attn_tc2_s200"] = lambda: check_attention(3, 200, 2, True, seed=12)
CHECKS["attn_tc2_s256_many"] = lambda: check_attention(20, 256, 4, True, seed=13)
CHECKS["attn_tc_drop_s128"] = lambda: check_attention(4, 128, 2, True, seed=14, dropout=0.1)
CHECKS["attn_tc2_drop_s200"] = lambda: check_attention(3, 200, 2, True, seed=15, dropout=0.1)
# 16 heads (H = 1024): the short (S <= 256) and key-blocked (S > 256) kernels
CHECKS["attn_h16_s128"] = lambda: check_attention(2, 128, 16, True, seed=80)
CHECKS["attn_h16_s256"] = lambda: check_attention(2, 256, 16, True, seed=81)
CHECKS["attn_h16_s512"] = lambda: check_attention(2, 512, 16, True, seed=82)
CHECKS["attn_h16_drop_s200"] = lambda: check_attention(2, 200, 16, True, seed=83, dropout=0.1)

# LayerNorm widths: H = 256 / 512 take the paired-column kernels at MAXC 1 / 2; H = 320 / 640 / 896 the generic kernels
# with a partly active last chunk (MAXC 2 / 3 / 4).  Each with and without the fp16 stream and the CLS-row output.
for _H in (256, 320, 512, 640, 896):
    CHECKS[f"ln_{_H}"] = lambda H=_H: check_ln(777, H, seed=H)
    CHECKS[f"ln_{_H}_f16"] = lambda H=_H: check_ln(777, H, seed=H + 1, f16=True)
    CHECKS[f"ln_{_H}_cls"] = lambda H=_H: check_ln(640, H, cls_stride=40, seed=H + 2)
    CHECKS[f"ln_{_H}_cls_f16"] = lambda H=_H: check_ln(640, H, cls_stride=40, seed=H + 3, f16=True)

# embeddings: dropout, the fp16 y_res copy, one and three token types, RoBERTa positions; T = 9000 rows (> 4224 warps)
for _H in (256, 320, 768, 1024):
    CHECKS[f"embed_{_H}_drop_yres_tt3"] = lambda H=_H: check_embed(9000, H, type_vocab=3, seed=H, dropout=0.1,
                                                                   y_res=True)
    CHECKS[f"embed_{_H}_roberta_tt1"] = lambda H=_H: check_embed(9000, H, type_vocab=1, seed=H + 1, y_res=True,
                                                                 dropout=0.1 if H in (320, 1024) else 0.0,
                                                                 roberta_S=100)


# ------------------------------------------------------------------ retrieval
def _r16(x):
    """float64 -> fp16 value (as float64), rounded through fp32.  Every score the kernel rounds is an fp32 value v with
    fl32(e - tol) <= v <= fl32(e + tol), and rounding is monotone, so bounds taken this way hold for its fp16 scores."""
    return x.float().half().double()


def check_search(Q=100, N=5000, d=768, k=100, bf16=False, seed=20, mode="random", offset=0, reference_ranking=False):
    """dprb_search_topk vs oracle/retrieval.py (restating run_retrieval_pytorch.py:141-176) on float64 scores.

    The float64 scores of the 16-bit operands (products of 16-bit values are exact in double) are computed on the GPU,
    a block of queries at a time, and ranked like oracle/retrieval.topk_desc (descending, ties by ascending row id).
    Tolerance: the kernel ranks by fp32-accumulated products of the identical 16-bit operands, so a returned score
    may differ from the float64 score e of the same row by tol = 1e-5 * max_row(|q|.|c|).
      * always: ids in range and distinct per query; scores non-increasing; equal scores in ascending id order.
      * default ranking: |returned - e| <= tol; ids agree with the oracle wherever scores are separated by more than
        2 tol, and the returned set is a valid top-k up to 2 tol.
      * reference_ranking (the fp16-rounded score, r16): a returned score h of a row lies in
        [r16(e - tol), r16(e + tol)].  A row is certain when r16(e - tol) == r16(e + tol): its fp16 score is known.  A certain row must be returned
        when that score is above the k-th returned score, or equal to it with an id below the largest returned id at
        that score.
    Modes with a known answer are checked exactly: "constant" (identical rows), "signed_zero_f16" and "zero_query"
    (every score is zero, -0 or +0) return rows 0..k-1 with one score.
    """
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(Q, d, generator=g)
    if mode == "random":
        c = torch.randn(N, d, generator=g)
    elif mode == "dup":          # every row appears twice -> exact score ties, resolved towards the lower id
        h = torch.randn((N + 1) // 2, d, generator=g)
        c = torch.cat([h, h], 0)[:N]
    elif mode == "ascending":    # scores grow with the row id for every query: worst case for the running threshold
        v = torch.randn(d, generator=g)
        q = q * 0.05 + v
        c = v[None, :] * (0.25 + torch.arange(N, dtype=torch.float32)[:, None] / N)
    elif mode == "descending":   # the best rows come first: the bar is final after the first tile
        v = torch.randn(d, generator=g)
        q = q * 0.05 + v
        c = v[None, :] * (1.25 - torch.arange(N, dtype=torch.float32)[:, None] / N)
    elif mode == "constant":     # every row identical: all scores tie, the answer is rows 0..k-1 for every query
        c = torch.randn(1, d, generator=g).expand(N, d).contiguous()
    elif mode == "negative":     # every score below 0
        q = q.abs() + 0.1
        c = -(torch.randn(N, d, generator=g).abs() + 0.1)
    elif mode == "signed_zero_f16":
        # q . c = +-2^-26 exactly in fp32; rounded to fp16 (below half the least subnormal 2^-24) every score is -0
        # (even rows) or +0 (odd rows): all equal, so the answer is rows 0..k-1
        assert reference_ranking, "signed_zero_f16 ranks by the fp16-rounded score"
        q = torch.zeros(Q, d)
        q[:, 0] = 2.0 ** -12
        c = torch.zeros(N, d)
        c[:, 0] = 2.0 ** -14 * (1.0 - 2.0 * (torch.arange(N) % 2 == 0).float())
    elif mode == "zero_query":   # zero queries: every score is 0 (a sum of -0 products against the all-negative rows)
        q = torch.zeros(Q, d)
        c = torch.randn(N, d, generator=g)
        c[::3] = -(c[::3].abs() + 0.1)
    else:
        raise ValueError(mode)
    dt = torch.bfloat16 if bf16 else torch.float16
    q16, c16 = q.to(dt).to(DEV), c.to(dt).to(DEV)
    s, i = ops.search_topk(q16, c16, k, index_offset=offset, reference_ranking=reference_ranking)
    torch.cuda.synchronize()
    assert s.shape == (Q, k) and i.shape == (Q, k)
    s, i = s.double(), i - offset
    assert bool(((i >= 0) & (i < N)).all()), "row ids out of range"
    assert bool((i.sort(1).values.diff(1) != 0).all()), "duplicate row ids"
    ds = s.diff(1)
    assert bool((ds <= 0).all()), "scores not descending"
    assert bool((i.diff(1)[ds == 0] > 0).all()), "equal scores not ordered by ascending row id"
    if mode in ("constant", "signed_zero_f16", "zero_query"):
        assert torch.equal(i, torch.arange(k, device=DEV).expand(Q, k)), "tied rows not returned as 0..k-1"
        assert bool((s == s[:, :1]).all()), "tied rows returned with different scores"
        if mode != "constant":
            assert bool((s == 0).all()), "zero scores returned as nonzero"

    qe, ce = q16.double(), c16.double()
    QC = max(1, (1 << 25) // N)          # float64 score blocks of <= 256 MB
    tol = 1e-5 * max(float((qe[a:a + QC].abs() @ ce.abs().T).max()) for a in range(0, Q, QC))
    out = {"tol": tol}
    maxerr = 0.0
    mism = certain = 0
    rows = torch.arange(N, device=DEV)
    for a in range(0, Q, QC):
        exact = qe[a:a + QC] @ ce.T
        sb, ib = s[a:a + QC], i[a:a + QC]
        got = exact.gather(1, ib)
        returned = torch.zeros_like(exact, dtype=torch.bool).scatter_(1, ib, True)
        if reference_ranking:
            assert bool(((_r16(got - tol) <= sb) & (sb <= _r16(got + tol))).all()), \
                "fp16 score outside [r16(e - tol), r16(e + tol)]"
            lo16 = _r16(exact - tol)
            sure = lo16 == _r16(exact + tol)
            hk = sb[:, -1:]
            last = torch.where(sb == hk, ib, -1).max(1, keepdim=True).values
            must = sure & ((lo16 > hk) | ((lo16 == hk) & (rows[None, :] < last)))
            assert bool(returned[must].all()), "missing a row whose fp16 score is certain to rank in the top-k"
            certain += int(sure.sum())
            continue
        maxerr = max(maxerr, float((got - sb).abs().max()))
        assert maxerr <= tol, f"score error {maxerr:.3e} > {tol:.3e}"
        os_, oi = exact.sort(dim=1, descending=True, stable=True)
        os_, oi = os_[:, :k + 1], oi[:, :k + 1]
        kth = os_[:, k - 1:k]
        assert bool((got >= kth - 2 * tol).all()), "returned a row that is not in the top-k"
        must = os_[:, :k] > kth + 2 * tol
        assert bool(returned.gather(1, oi[:, :k])[must].all()), "missing rows with score above the k-th"
        inf = torch.full_like(kth, math.inf)
        gap = os_[:, :-1] - os_[:, 1:]                        # gap[:, j] = e[j] - e[j + 1]
        lo = torch.cat([gap, inf], 1)[:, :k]
        hi = torch.cat([inf, gap], 1)[:, :k]
        sep = (lo > 2 * tol) & (hi > 2 * tol)
        same = ib == oi[:, :k]
        assert bool(same[sep].all()), "ids differ from the oracle where scores are separated by more than 2 tol"
        mism += int((~same & ~sep).sum())
    if reference_ranking:
        out["certain_rows"] = certain
    else:
        out["score_maxerr"] = maxerr
        out["near_tie_swaps"] = mism
    return out


def check_topk_merge(Q=37, total=300, k=100, seed=30, signed_zero=False):
    """dprb_topk_merge vs the restated shard merge (run_retrieval_pytorch.py:272-277: topk over the concatenated shard
    results + gather); bit-exact (fp32 compare / select only), ties towards the earlier position.
    signed_zero: -0.0 at even and +0.0 at odd positions, all equal scores, so the answer is positions 0..k-1."""
    import numpy as np
    from oracle import retrieval as R
    g = torch.Generator().manual_seed(seed)
    s = torch.randn(Q, total, generator=g)
    nt = min(s[:, ::7].shape[1], s[:, 3::7].shape[1])
    s[:, 0:7 * nt:7] = s[:, 3:3 + 7 * nt:7]                  # inject exact ties
    if signed_zero:
        s = torch.zeros(Q, total)
        s[:, 0::2] = -0.0
    idx = torch.randint(0, 2 ** 40, (Q, total), generator=g, dtype=torch.int64)
    ms, mi = ops.topk_merge(s.to(DEV), idx.to(DEV), k)
    torch.cuda.synchronize()
    rs, order = R.topk_desc(s.numpy().astype(np.float64), k)
    if signed_zero:
        assert np.array_equal(order, np.broadcast_to(np.arange(k), (Q, k)))
    ri = np.take_along_axis(idx.numpy(), order, axis=1)
    assert np.array_equal(ms.cpu().numpy().astype(np.float64), rs), "merged scores differ"
    assert np.array_equal(mi.cpu().numpy(), ri), "merged ids differ"
    return {"exact": True}


CHECKS["search_fp16_100x5000"] = lambda: check_search(100, 5000, 768, 100)
CHECKS["search_small_ragged"] = lambda: check_search(7, 1000, 200, 10, seed=21)
CHECKS["search_k_equals_n_region"] = lambda: check_search(5, 300, 64, 256, seed=22)
CHECKS["search_one_query_k1"] = lambda: check_search(1, 4097, 128, 1, seed=23)
CHECKS["search_bf16_300x70000"] = lambda: check_search(300, 70000, 1024, 256, bf16=True, seed=24, offset=1000000)
CHECKS["search_many_query_tiles"] = lambda: check_search(1100, 30000, 256, 100, seed=25)
CHECKS["search_k1000"] = lambda: check_search(40, 60000, 128, 1000, seed=26)
CHECKS["search_duplicate_rows"] = lambda: check_search(33, 9000, 128, 50, seed=27, mode="dup")
CHECKS["search_ascending_scores"] = lambda: check_search(64, 20000, 64, 100, seed=28, mode="ascending")
CHECKS["search_all_equal"] = lambda: check_search(40, 5000, 64, 100, seed=29, mode="constant")
CHECKS["topk_merge"] = lambda: check_topk_merge()
CHECKS["topk_merge_large"] = lambda: check_topk_merge(Q=5, total=40000, k=1000, seed=31)
