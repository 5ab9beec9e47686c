"""Host-side pieces of the encoder stage tests (test_encoder_stages_gpu): the restated workspace carve of encoder.cu's
plan(), held to dprb_encoder_workspace_bytes (a host-only entry point: the library loads without a device), and the
fitted-CDF GELU errors the GEMM epilogues document, confirmed on a float64 restatement of gelu_and_grad2."""
import ctypes
import itertools
import math

import torch

# common.cuh documents max |x Phi_fit - gelu_erf| 3.0e-5 and a derivative error of 1.2e-4 (rounded: 1.211e-4 on the
# grid of test_gelu_fit_error_bounds_cpu)
GELU_FIT, DGELU_FIT = 3.0e-5, 1.25e-4


def _nbytes(dtype, shape):
    return math.prod(shape) * (2 if dtype in (torch.bfloat16, torch.float16) else 4)


def layout(H, I, L, heads, nseq, S, save):
    """({key: (byte offset, dtype, shape)}, total bytes) of plan()'s carve.  Per-layer keys are (name, slot); save = 0
    keeps two slots (layer l in slot l & 1); save = 2 (lean) points every slot's ctx / hact at one shared buffer.
    Carve rounds every buffer up to 256 bytes."""
    T = nseq * S
    off, lay = 0, {}
    bf, f16, f32 = torch.bfloat16, torch.float16, torch.float32

    def take(key, dtype, shape):
        nonlocal off
        lay[key] = (off, dtype, shape)
        off += (_nbytes(dtype, shape) + 255) // 256 * 256

    take("rA", f16, (T, H))
    take("rB", f16, (T, H))
    take("x0", bf, (T, H))
    take("emb_stats", f32, (T, 2))
    lean = save == 2
    if lean:
        take("ctx_t", bf, (T, H))
        take("hact_t", bf, (T, I))
    for s in range(L if save else 2):
        take(("qkv", s), bf, (T, 3 * H))
        if lean:
            lay[("ctx", s)] = lay["ctx_t"]
        else:
            take(("ctx", s), bf, (T, H))
        take(("lse", s), f32, (nseq * heads * S,))
        take(("z1", s), f16, (T, H))
        take(("stats1", s), f32, (T, 2))
        take(("x1", s), bf, (T, H))
        if save:
            take(("hpre", s), bf, (T, I))
        if lean:
            lay[("hact", s)] = lay["hact_t"]
        else:
            take(("hact", s), bf, (T, I))
        take(("z2", s), f16, (T, H))
        take(("stats2", s), f32, (T, 2))
        take(("out", s), bf, (T, H))
    if save:
        for name, width in (("gA", H), ("gB", H), ("gB2", H), ("gH", I), ("gQKV", 3 * H)):
            take(name, bf, (T, width))
    return lay, off


def views(ws, base_ptr, lay):
    """Typed views of the workspace tensor `ws` (uint8) at the 256-aligned base the library was handed."""
    b0 = base_ptr - ws.data_ptr()
    return {key: ws[b0 + off:b0 + off + _nbytes(dtype, shape)].view(dtype).view(shape)
            for key, (off, dtype, shape) in lay.items()}


def gelu_fit64(x):
    """float64 restatement of common.cuh gelu_and_grad2: (x sigma(z(x)), its derivative), z's argument clamped at
    x^2 = 64."""
    x2 = torch.clamp(x * x, max=64.0)
    pz = (x2 * 1.03455483e-3 - 1.06900513e-1) * x2 - 2.30098511
    sg = 1.0 / (1.0 + torch.exp2(pz * x))
    zp = (x2 * -3.58549371e-3 + 2.22293380e-1) * x2 + 1.59492135
    return x * sg, sg * (x * (1.0 - sg) * zp + 1.0)


def gelu64(x):
    """erf-GELU and its derivative."""
    cdf = 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0)))
    return x * cdf, cdf + x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)


def test_workspace_layout_matches_the_library_cpu():
    """The restated carve has the library's size over a grid of shapes and the three save modes: a change to plan()
    fails here instead of misreading buffers in the stage tests."""
    from dpr_scale_b200 import _lib
    lib = _lib.load()
    n = 0
    for (H, heads), I, L, nseq, S, save in itertools.product(((128, 2), (320, 5), (768, 12), (1024, 16)),
                                                           (512, 1288, 3072, 4096), (1, 2, 3, 12), (1, 3, 7),
                                                           (1, 37, 128, 200, 512), (0, 1, 2)):
        w = _lib.EncoderWeights()
        w.hidden, w.inter, w.layers, w.heads = H, I, L, heads
        want = lib.dprb_encoder_workspace_bytes(ctypes.byref(w), nseq, S, save)
        assert layout(H, I, L, heads, nseq, S, save)[1] == want, (H, I, L, heads, nseq, S, save)
        n += 1
    print(f"{n} shapes: restated layout == dprb_encoder_workspace_bytes")


def test_workspace_layout_buffers_are_disjoint_and_aligned_cpu():
    """Every buffer starts 256-byte aligned and, apart from lean mode's shared ctx / hact, no two overlap."""
    for save in (0, 1, 2):
        lay, total = layout(320, 1288, 3, 5, 7, 37, save)
        spans = sorted({(off, off + _nbytes(dt, shape)) for off, dt, shape in lay.values()})
        assert all(a % 256 == 0 for a, _ in spans) and spans[-1][1] <= total
        assert all(spans[i][1] <= spans[i + 1][0] for i in range(len(spans) - 1)), save


def test_gelu_fit_error_bounds_cpu():
    """The fitted-CDF errors the GELU epilogues document hold on a fine grid (the stage tests' GELU gates use them)."""
    x = torch.linspace(-20.0, 20.0, 2_000_001, dtype=torch.float64)
    g, d = gelu_fit64(x)
    gr, dr = gelu64(x)
    eg, ed = float((g - gr).abs().max()), float((d - dr).abs().max())
    print(f"gelu fit: max |g err| {eg:.3g}, max |g' err| {ed:.3g}")
    assert eg <= GELU_FIT and ed <= DGELU_FIT
