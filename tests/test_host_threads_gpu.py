"""The C entry points may be called from any host thread (INTEGRATION.md, "Ownership and threading"): autograd runs
backward on its own thread, where a library call may be the first CUDA call of any kind.  Every buffer is allocated
on the main thread; a fresh thread then calls the C ABI directly (no torch call inside it) and must get the same
return codes and bit-identical outputs as the same calls made on the main thread."""
import threading

import pytest
import torch

pytestmark = pytest.mark.gpu


def _problem():
    g = torch.Generator().manual_seed(11)
    r = lambda *s, dt=torch.float32: (torch.randn(*s, generator=g) * 0.5).to(dt).cuda()
    x = {"A": r(256, 256, dt=torch.bfloat16), "B": r(512, 256, dt=torch.bfloat16), "bias": r(512),
         "q": r(128, 128), "c": r(256, 128), "labels": torch.randint(0, 256, (128,), generator=g).cuda(),
         "queries": r(300, 128, dt=torch.float16), "corpus": r(5000, 128, dt=torch.float16)}
    for S in (128, 384):     # the S <= 256 kernels and the 256 < S <= 512 kernels; 2 sequences x 2 heads
        x[f"qkv{S}"], x[f"dctx{S}"] = r(2 * S, 384, dt=torch.bfloat16), r(2 * S, 128, dt=torch.bfloat16)
    return x


def _outputs(lib):
    """Output buffers (NaN-filled, so that an unwritten element fails the comparison) and workspaces."""
    e = lambda *s, dt=torch.float32: torch.full(s, float("nan"), dtype=dt, device="cuda")
    o = {"D": e(256, 512, dt=torch.bfloat16), "score_lse": e(128), "dq": e(128, 128), "dc": e(256, 128),
         "scores": e(300, 10), "index": torch.zeros(300, 10, dtype=torch.int64, device="cuda")}
    for S in (128, 384):
        o[f"ctx{S}"], o[f"lse{S}"] = e(2 * S, 128, dt=torch.bfloat16), e(2, 2, S)
        o[f"dqkv{S}"] = e(2 * S, 384, dt=torch.bfloat16)
    ws = {"score": int(lib.dprb_score_tc_workspace_bytes(128, 256, 128, 128, 256)),
          "search": int(lib.dprb_search_workspace_bytes(300, 10))}
    assert min(ws.values()) > 0
    return o, {k: torch.empty(n, dtype=torch.uint8, device="cuda") for k, n in ws.items()}


def _families(lib, x, o, ws):
    """Each entry-point family as a callable returning {name: rc}, on the legacy default stream.  Only ctypes and
    data_ptr() in here."""
    p = lambda t: t.data_ptr()

    def gemm():   # EPI_BIAS, no split-K
        return {"gemm": lib.dprb_gemm_bf16(p(x["A"]), p(x["B"]), p(o["D"]), 256, 512, 256, 256, 256, 512, 0, 0, 0,
                                           p(x["bias"]), None, 0, None, 1.0, 1, None, 0.0, 0, None)}

    def attention(S):
        qkv, ctx, lse = p(x[f"qkv{S}"]), p(o[f"ctx{S}"]), p(o[f"lse{S}"])
        return {f"attn_fwd{S}": lib.dprb_attn_fwd(qkv, None, ctx, lse, 2, S, 2, 0.0, 0, None),
                f"attn_bwd{S}": lib.dprb_attn_bwd(qkv, None, ctx, lse, p(x[f"dctx{S}"]), p(o[f"dqkv{S}"]), None, 2, S,
                                                  2, 0.0, 0, None)}

    def score():   # no loss_sum: it is an fp32 atomicAdd over warps, so its last bit depends on their order
        w = ws["score"]
        return {"score_fwd": lib.dprb_score_tc_fwd(p(x["q"]), p(x["c"]), None, None, p(x["labels"]), 20.0,
                                                   p(o["score_lse"]), None, None, 128, 256, 128, 128, 256, p(w),
                                                   w.numel(), None),
                "score_bwd": lib.dprb_score_tc_bwd(None, None, p(x["labels"]), p(o["score_lse"]), 1.0, 20.0, p(o["dq"]),
                                                   p(o["dc"]), 128, 256, 128, 0, 128, 0, 256, p(w), w.numel(), None)}

    def search():
        w = ws["search"]
        return {"search": lib.dprb_search_topk(p(x["queries"]), p(x["corpus"]), 0, 300, 5000, 128, 10, 0,
                                               p(o["scores"]), p(o["index"]), p(w), w.numel(), None)}

    return {"gemm": gemm, "attention128": lambda: attention(128), "attention384": lambda: attention(384),
            "score": score, "search": search}


@pytest.mark.parametrize("family", ["gemm", "attention128", "attention384", "score", "search"])
def test_entry_points_from_a_fresh_thread(family):
    """The family's calls are the first CUDA calls of their thread: nothing else has bound a context there."""
    from dpr_scale_b200 import _lib
    lib = _lib.load()
    x = _problem()
    (main_out, main_ws), (thread_out, thread_ws) = _outputs(lib), _outputs(lib)
    torch.cuda.synchronize()
    want = _families(lib, x, main_out, main_ws)[family]()
    assert want == {k: 0 for k in want}, lib.dprb_last_error()
    torch.cuda.synchronize()
    got = {}

    def worker():
        got.update(_families(lib, x, thread_out, thread_ws)[family]())
        got["error"] = lib.dprb_last_error()          # thread-local

    t = threading.Thread(target=worker)
    t.start()
    t.join()
    error = got.pop("error", None)
    assert got == want, error
    torch.cuda.synchronize()
    for name in {"gemm": ["D"], "attention128": ["ctx128", "lse128", "dqkv128"],
                 "attention384": ["ctx384", "lse384", "dqkv384"], "score": ["score_lse", "dq", "dc"],
                 "search": ["scores", "index"]}[family]:
        a, b = main_out[name], thread_out[name]
        if a.is_floating_point():
            assert not torch.isnan(a).any(), f"{name}: output not written"
            a, b = a.view(torch.uint8), b.view(torch.uint8)
        assert torch.equal(a, b), f"{name} differs between threads"
