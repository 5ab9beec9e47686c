"""GEMM cases that exercise the persistent scheduler: more work units than SMs (each CTA walks several tiles and the
smem ring runs across tile boundaries), partial 128x256 tiles in M and N, and split-K unit counts that do not divide
evenly over the grid."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _check_residual_dropout(M, N, K, p=0.1, seed=7):
    """EPI_BIAS_RESIDUAL with hidden dropout and the fused column sums: D = dropout(A B^T + bias) + aux, against the
    oracle's (row, col, site seed) keep mask."""
    from dpr_scale_b200 import ops
    from oracle import dropout as odrop
    from tests.gpu_checks import _bf, _close
    g = torch.Generator().manual_seed(seed)
    A = _bf(torch.randn(M, K, generator=g))
    B = _bf(torch.randn(N, K, generator=g) * 0.5)
    bias = torch.randn(N, generator=g)
    aux = _bf(torch.randn(M, N, generator=g))
    site = odrop.site_seed32(1234, 3, 2)
    out = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    cs = torch.zeros(N, device="cuda")
    ops.gemm(A.cuda(), B.cuda(), out, M, N, K, K, K, N, False, False, ops.EPI_BIAS_RESIDUAL, bias.cuda(), aux.cuda(), N,
             colsum=cs, dropout_p=p, drop_seed=site)
    torch.cuda.synchronize()
    keep = torch.from_numpy(odrop.keep_mask(M, N, p, 1234, 3, 2)).double()
    want = (A.double() @ B.double().T + bias.double()) * keep * odrop.scale(p) + aux.double()
    res = {}
    _close("gemm_drop_res", out, want, 2 ** -7, 1e-3, res)
    _close("gemm_drop_res_colsum", cs, out.double().cpu().sum(0), 1e-5, 1e-3, res)
    return res


def _cases():
    from dpr_scale_b200 import ops
    from tests.gpu_checks import check_gemm, check_gemm_f16_stream, check_gemm_lean
    return {
        # 32 x 9 = 288 units: more than one per SM for every epilogue
        "many_units_bias": lambda: check_gemm(4096, 2304, 256),
        "many_units_residual": lambda: check_gemm(4096, 2304, 256, epilogue=ops.EPI_BIAS_RESIDUAL),
        "many_units_gelu": lambda: check_gemm(4096, 2304, 256, epilogue=ops.EPI_BIAS_GELU),
        "many_units_dgelu": lambda: check_gemm(4096, 2304, 256, b_mn=True, epilogue=ops.EPI_DGELU),
        "many_units_f32_store": lambda: check_gemm(4096, 2304, 256, epilogue=ops.EPI_F32_STORE),
        "many_units_atomic": lambda: check_gemm(4096, 2304, 256, a_mn=True, b_mn=True, epilogue=ops.EPI_F32_ATOMIC_ADD),
        "many_units_lean": lambda: check_gemm_lean(4096, 2304, 256, seed=42),
        "many_units_f16_stream": lambda: check_gemm_f16_stream(4096, 2304, 256, seed=32),
        # N not a multiple of 256, M not a multiple of 128, with dropout + residual + column sums
        "drop_res_n520": lambda: _check_residual_dropout(300, 520, 200),
        "drop_res_n264": lambda: _check_residual_dropout(1000, 264, 192, seed=8),
        "drop_res_many_units": lambda: _check_residual_dropout(8200, 776, 128, seed=9),
        "m_ragged_residual": lambda: check_gemm(1000, 768, 512, epilogue=ops.EPI_BIAS_RESIDUAL),
        "m_ragged_dgelu_colsum": lambda: check_gemm(77, 264, 128, b_mn=True, epilogue=ops.EPI_DGELU),
        "m_ragged_mn_a": lambda: check_gemm(200, 520, 320, a_mn=True),
        # split-K: 18 tiles x 5 splits = 90 units (fewer than the SMs); 32 tiles x 6 splits = 192 (not a multiple)
        "splitk_partial_grid": lambda: check_gemm(768, 768, 2048, a_mn=True, b_mn=True, epilogue=ops.EPI_F32_ATOMIC_ADD,
                                                  splits=5),
        "splitk_uneven_units": lambda: check_gemm(1000, 1000, 1000, a_mn=True, b_mn=True,
                                                  epilogue=ops.EPI_F32_ATOMIC_ADD, splits=7),
        "splitk_auto_tall_k": lambda: check_gemm(768, 3072, 16384, a_mn=True, b_mn=True, epilogue=ops.EPI_F32_ATOMIC_ADD,
                                                 splits=0),
    }


@pytest.mark.parametrize("name", sorted(_cases()))
def test_gemm_schedule(name):
    res = _cases()[name]()
    assert res, name
