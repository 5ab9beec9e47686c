"""16-bit GEMM epilogues through the TMA-staged slab: every epilogue with more work units than two per SM (each CTA hands
its staging slab between the producer's aux load and the consumers' TMA stores several times), partial tiles that TMA
must clip on store and zero-fill on load, strided aux / D / out2, and a guard band around every output that must stay
untouched."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

GUARD_ROWS = 64          # a whole warpgroup slab of rows past M
GUARD_COLS = 72          # past N: more than the 64-column box that straddles N


def _guarded(M, N, ld, dtype, g):
    """A [M + GUARD_ROWS, ld] buffer of random bits and its [M, N] view with leading dimension ld."""
    buf = torch.randn(M + GUARD_ROWS, ld, generator=g).to(dtype).cuda()
    return buf, buf[:M, :N]


def _untouched(name, before, after, M, N):
    outside = torch.ones(before.shape, dtype=torch.bool)
    outside[:M, :N] = False
    b = before.cpu().view(torch.int16)[outside]
    a = after.cpu().view(torch.int16)[outside]
    assert torch.equal(a, b), f"{name}: {int((a != b).sum())} elements written outside [{M}, {N}]"


def _gelu_grad(x):
    cdf = 0.5 * (1 + torch.erf(x / math.sqrt(2)))
    return cdf + x * torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)


def _check(M, N, K, epi, *, b_mn=False, colsum=False, drop=0.0, out2=False, lean=False, f16=False, strided=False,
           seed=0):
    from dpr_scale_b200 import ops
    from oracle import dropout as odrop
    from oracle import encoder as oenc
    from tests.gpu_checks import _bf, _close
    g = torch.Generator().manual_seed(seed)
    A = _bf(torch.randn(M, K, generator=g))
    B = _bf(torch.randn(N, K, generator=g) * 0.3)
    bias = torch.randn(N, generator=g)
    aux_dt = torch.float16 if f16 else torch.bfloat16
    aux = (torch.randn(M, N, generator=g) * (3 if f16 else 1)).to(aux_dt)
    ldd = N + GUARD_COLS if strided else N
    ld_aux = N + 40 if strided else N
    aux_buf = torch.randn(M, ld_aux, generator=g).to(aux_dt)
    aux_buf[:, :N] = aux
    aux_d = aux_buf.cuda()[:, :N]
    out_buf, out = _guarded(M, N, ldd, torch.float16 if f16 else torch.bfloat16, g)
    out_before = out_buf.clone()
    o2_buf, o2 = _guarded(M, N, ldd, torch.bfloat16, g) if out2 else (None, None)
    o2_before = o2_buf.clone() if out2 else None
    cs = torch.zeros(N, device="cuda") if colsum else None

    flags = (ops.GEMM_SAVE_PRE if lean else 0) | ((ops.GEMM_AUX_F16 | ops.GEMM_OUT_F16) if f16 else 0)
    use_aux = epi in (ops.EPI_BIAS_RESIDUAL, ops.EPI_DGELU, ops.EPI_DGELU_PRE)
    use_bias = epi in (ops.EPI_BIAS, ops.EPI_BIAS_GELU, ops.EPI_BIAS_RESIDUAL)
    site = odrop.site_seed32(99, 1, 3)
    Bd = (B.T.contiguous() if b_mn else B).cuda()
    ops.gemm(A.cuda(), Bd, out, M, N, K, K, N if b_mn else K, ldd, False, b_mn, epi | flags,
             bias.cuda() if use_bias else None, aux_d if use_aux else None, ld_aux if use_aux else 0, o2, colsum=cs,
             dropout_p=drop, drop_seed=site if drop else 0)
    torch.cuda.synchronize()

    acc = A.double() @ B.double().T
    res = {}
    if epi == ops.EPI_BIAS_GELU:
        pre = acc + bias.double()
        want = oenc.gelu_erf(pre)
        if out2:
            _close("out2", o2, pre if lean else _gelu_grad(pre), 2 ** -7, 1e-3, res)
    elif epi == ops.EPI_BIAS_RESIDUAL:
        v = acc + bias.double()
        if drop:
            v = v * torch.from_numpy(odrop.keep_mask(M, N, drop, 99, 1, 3)).double() * odrop.scale(drop)
        want = v + aux.double()
    elif epi == ops.EPI_DGELU:
        want = acc * aux.double()
    elif epi == ops.EPI_DGELU_PRE:
        want = acc * _gelu_grad(aux.double())
    else:
        want = acc + bias.double()
    _close("out", out, want, 2 ** -10 if f16 else 2 ** -7, 2e-3, res)
    if colsum:
        _close("colsum", cs, out.double().cpu().sum(0), 1e-5, 1e-3, res)
    _untouched("out", out_before, out_buf, M, N)
    if out2:
        _untouched("out2", o2_before, o2_buf, M, N)
    return res


def _cases():
    from dpr_scale_b200 import ops
    E = ops
    # 32 x 9 = 288 units of 128 x 256 on 132 SMs: every CTA runs at least two tiles through its slab
    big = (4096, 2304, 128)
    return {
        "bias": lambda: _check(*big, E.EPI_BIAS),
        "bias_colsum": lambda: _check(*big, E.EPI_BIAS, colsum=True, b_mn=True),
        "gelu": lambda: _check(*big, E.EPI_BIAS_GELU),
        "gelu_out2": lambda: _check(*big, E.EPI_BIAS_GELU, out2=True),
        "gelu_lean": lambda: _check(*big, E.EPI_BIAS_GELU, out2=True, lean=True),
        "residual": lambda: _check(*big, E.EPI_BIAS_RESIDUAL),
        "residual_drop": lambda: _check(*big, E.EPI_BIAS_RESIDUAL, drop=0.1),
        "residual_drop_colsum": lambda: _check(*big, E.EPI_BIAS_RESIDUAL, drop=0.1, colsum=True),
        "residual_colsum_mn": lambda: _check(*big, E.EPI_BIAS_RESIDUAL, colsum=True, b_mn=True),
        "dgelu_colsum": lambda: _check(*big, E.EPI_DGELU, colsum=True, b_mn=True),
        "dgelu_pre_colsum": lambda: _check(*big, E.EPI_DGELU_PRE, colsum=True, b_mn=True),
        "f16_residual": lambda: _check(*big, E.EPI_BIAS_RESIDUAL, f16=True),
        "f16_residual_drop": lambda: _check(*big, E.EPI_BIAS_RESIDUAL, f16=True, drop=0.1),
        # one k-block per unit: the slab is released and refilled around a single MMA step
        "one_kblock_residual": lambda: _check(4096, 2304, 64, E.EPI_BIAS_RESIDUAL, colsum=True),
        # partial tiles: M % 128 != 0, N % 64 != 0 (N % 8 == 0), clipped on store and zero-filled on load
        "ragged_residual_drop": lambda: _check(1000, 328, 192, E.EPI_BIAS_RESIDUAL, drop=0.1, colsum=True, strided=True),
        "ragged_gelu_out2": lambda: _check(1000, 200, 128, E.EPI_BIAS_GELU, out2=True, strided=True),
        "ragged_dgelu_pre": lambda: _check(1000, 584, 256, E.EPI_DGELU_PRE, colsum=True, b_mn=True, strided=True),
        "ragged_f16": lambda: _check(3000, 776, 128, E.EPI_BIAS_RESIDUAL, f16=True, strided=True),
        "single_tile_m77": lambda: _check(77, 264, 128, E.EPI_DGELU, colsum=True, b_mn=True, strided=True),
        "single_tile_m40_bias": lambda: _check(40, 136, 64, E.EPI_BIAS, strided=True),
        # the pruned last layer: a few CLS rows whose residual rows are S * H apart
        "strided_aux_many_units": lambda: _check(4096, 2304, 128, E.EPI_BIAS_RESIDUAL, drop=0.1, strided=True),
    }


@pytest.mark.parametrize("name", sorted(_cases()))
def test_gemm_epilogue(name):
    res = _cases()[name]()
    assert res, name


def test_pruned_layer_residual_stride():
    """The pruned last layer's attention-output GEMM: R = nseq rows, residual read with ld_aux = S * H from the full
    [T, H] fp16 stream, D written densely."""
    from dpr_scale_b200 import ops
    from tests.gpu_checks import _bf, _close
    nseq, S, H = 300, 128, 768
    g = torch.Generator().manual_seed(5)
    A = _bf(torch.randn(nseq, H, generator=g))
    W = _bf(torch.randn(H, H, generator=g) * 0.05)
    bias = torch.randn(H, generator=g)
    stream = (torch.randn(nseq * S, H, generator=g) * 3).half()
    out_buf, out = _guarded(nseq, H, H, torch.float16, g)
    before = out_buf.clone()
    ops.gemm(A.cuda(), W.cuda(), out, nseq, H, H, H, H, H, False, False,
             ops.EPI_BIAS_RESIDUAL | ops.GEMM_AUX_F16 | ops.GEMM_OUT_F16, bias.cuda(), stream.cuda(), S * H)
    torch.cuda.synchronize()
    want = A.double() @ W.double().T + bias.double() + stream[::S].double()
    res = {}
    _close("pruned_residual", out, want, 2 ** -10, 2e-3, res)
    _untouched("pruned_residual", before, out_buf, nseq, H)
