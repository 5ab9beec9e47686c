"""Tensor-level wrappers over the C ABI (raw device pointers + the current CUDA stream).

PyTorch is plumbing here: device memory, streams, autograd bookkeeping.  Every function launches
hand-written sm_90a kernels from libdprb.so; nothing falls back to torch math.
"""
import ctypes

import numpy as np
import torch

from . import _lib
from ._lib import check

EPI_BIAS, EPI_BIAS_GELU, EPI_BIAS_RESIDUAL, EPI_DGELU, EPI_F32_ATOMIC_ADD, EPI_F32_STORE, EPI_DGELU_PRE = range(7)
GEMM_SAVE_PRE = 0x1000
# OR-ed into the epilogue: that operand holds fp16 instead of bf16 (include/dprb.h DPRB_GEMM_*_F16)
GEMM_A_F16, GEMM_B_F16, GEMM_AUX_F16, GEMM_OUT_F16 = 0x100, 0x200, 0x400, 0x800

def launch_count():
    """Kernels launched by libdprb.so in this process so far (counted inside the C launchers)."""
    return int(_lib.load().dprb_launch_count())


def _ptr(t):
    if t is None:
        return None
    assert t.is_cuda, "dprb ops need CUDA tensors (no CPU fallback)"
    return t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def gemm(a, b, out, M, N, K, lda, ldb, ldd, a_mn=False, b_mn=False, epilogue=EPI_BIAS, bias=None, aux=None,
         ld_aux=0, out2=None, alpha=1.0, splits=1, colsum=None, dropout_p=0.0, drop_seed=0):
    lib = _lib.load()
    check(lib.dprb_gemm_bf16(_ptr(a), _ptr(b), _ptr(out), M, N, K, lda, ldb, ldd, int(a_mn), int(b_mn), epilogue,
                             _ptr(bias), _ptr(aux), ld_aux, _ptr(out2), float(alpha), splits, _ptr(colsum),
                             float(dropout_p), int(drop_seed), _stream()),
          "dprb_gemm_bf16")
    return out


def linear_fwd(x, w, bias=None, epilogue=EPI_BIAS, aux=None, out2=None):
    """y[T,N] = epi(x[T,K] @ w[N,K]^T + bias); x, w bf16 contiguous; bias fp32."""
    T, K = x.shape
    N = w.shape[0]
    y = torch.empty(T, N, dtype=torch.bfloat16, device=x.device)
    gemm(x, w, y, T, N, K, K, K, N, False, False, epilogue, bias, aux, N if aux is not None else 0, out2)
    return y


def embed_ln_fwd(ids, type_ids, pos_ids, word, pos, typ, gamma, beta, eps, dropout_p=0.0, seed=0, y_res=None):
    """y_res: optional fp16 [T, H] tensor that receives a second copy of the output (the residual-stream copy)."""
    T = ids.numel()
    H = word.shape[1]
    y = torch.empty(T, H, dtype=torch.bfloat16, device=word.device)
    stats = torch.empty(T, 2, dtype=torch.float32, device=word.device)
    check(_lib.load().dprb_embed_ln_fwd(_ptr(ids), _ptr(type_ids), _ptr(pos_ids), _ptr(word), _ptr(pos), _ptr(typ),
                                        _ptr(gamma), _ptr(beta), _ptr(y), _ptr(stats), T, H, word.shape[0],
                                        pos.shape[0], typ.shape[0], float(eps), float(dropout_p), int(seed), _ptr(y_res),
                                        _stream()), "dprb_embed_ln_fwd")
    return y, stats


def embed_ln_bwd(dy, ids, type_ids, pos_ids, word, pos, typ, gamma, stats, dword, dpos, dtyp, dgamma, dbeta,
                 dropout_p=0.0, seed=0):
    T = ids.numel()
    H = word.shape[1]
    check(_lib.load().dprb_embed_ln_bwd(_ptr(dy), _ptr(ids), _ptr(type_ids), _ptr(pos_ids), _ptr(word), _ptr(pos),
                                        _ptr(typ), _ptr(gamma), _ptr(stats), _ptr(dword), _ptr(dpos), _ptr(dtyp),
                                        _ptr(dgamma), _ptr(dbeta), T, H, float(dropout_p), int(seed), _stream()),
          "dprb_embed_ln_bwd")


def ln_fwd(z, gamma, beta, eps, cls_stride=0, y_res=None):
    """z: bf16, or fp16 (the encoder's residual-stream sums); y: bf16; y_res: optional fp16 copy of y."""
    T, H = z.shape
    y = torch.empty(T, H, dtype=torch.bfloat16, device=z.device)
    stats = torch.empty(T, 2, dtype=torch.float32, device=z.device)
    cls = None
    if cls_stride:
        cls = torch.empty((T + cls_stride - 1) // cls_stride, H, dtype=torch.float32, device=z.device)
    check(_lib.load().dprb_ln_fwd(_ptr(z), _ptr(gamma), _ptr(beta), _ptr(y), _ptr(stats), _ptr(cls),
                                  cls_stride if cls_stride else 1, T, H, float(eps), int(z.dtype == torch.float16),
                                  _ptr(y_res), _stream()), "dprb_ln_fwd")
    return y, stats, cls


def ln_bwd(dy, z, stats, gamma, dgamma, dbeta, dbias=None, dy_cls=None, cls_stride=1, dropout_p=0.0, site_seed=0,
           dz=None, dzm=None):
    """dz / dzm: optional preallocated bf16 [T, H] outputs."""
    T, H = z.shape
    if dz is None:
        dz = torch.empty(z.shape, dtype=torch.bfloat16, device=z.device)      # gradients are bf16 whatever z holds
    if dzm is None and dropout_p > 0:
        dzm = torch.empty_like(dz)
    check(_lib.load().dprb_ln_bwd(_ptr(dy), _ptr(dy_cls), cls_stride, _ptr(z), _ptr(stats), _ptr(gamma), _ptr(dz),
                                  _ptr(dgamma), _ptr(dbeta), _ptr(dbias), T, H, _ptr(dzm), float(dropout_p),
                                  int(site_seed), int(z.dtype == torch.float16), _stream()), "dprb_ln_bwd")
    return (dz, dzm) if dropout_p > 0 else dz


def dropout_site_seed(seed, layer, site):
    return int(_lib.load().dprb_dropout_site_seed(int(seed), layer, site))


def dropout_mask(rows, cols, p, seed, layer, site, device="cuda"):
    """keep mask (uint8 [rows, cols]) of one dropout site — test aid."""
    out = torch.empty(rows, cols, dtype=torch.uint8, device=device)
    check(_lib.load().dprb_dropout_mask(_ptr(out), rows, cols, float(p), int(seed), layer, site, _stream()),
          "dprb_dropout_mask")
    return out


def gelu_from_pre(pre):
    out = torch.empty_like(pre)
    check(_lib.load().dprb_gelu_from_pre(_ptr(pre), _ptr(out), pre.numel(), _stream()), "dprb_gelu_from_pre")
    return out


def colsum(x, out):
    T, N = x.shape
    check(_lib.load().dprb_colsum_bf16(_ptr(x), x.stride(0), _ptr(out), T, N, _stream()), "dprb_colsum_bf16")
    return out


def attn_fwd(qkv, attn_mask, nseq, S, heads, need_lse=True, dropout_p=0.0, site_seed=0, ctx=None, lse=None):
    """ctx bf16 [nseq*S, H], lse fp32 [nseq, heads, S] (ctx / lse: optional preallocated outputs; the kernels write
    the first nseq*S rows and nseq*heads*S values)."""
    T = nseq * S
    H = heads * 64
    if ctx is None:
        ctx = torch.empty(T, H, dtype=torch.bfloat16, device=qkv.device)
    if lse is None and need_lse:
        lse = torch.empty(nseq, heads, S, dtype=torch.float32, device=qkv.device)
    check(_lib.load().dprb_attn_fwd(_ptr(qkv), _ptr(attn_mask), _ptr(ctx), _ptr(lse), nseq, S, heads, float(dropout_p),
                                    int(site_seed), _stream()), "dprb_attn_fwd")
    return ctx, lse


def attn_bwd(qkv, attn_mask, ctx, lse, dctx, nseq, S, heads, dbias=None, dropout_p=0.0, site_seed=0, dqkv=None):
    """dqkv bf16 [nseq*S, 3H] (dqkv: optional preallocated output; the first nseq*S rows are written)."""
    if dqkv is None:
        dqkv = torch.empty_like(qkv)
    check(_lib.load().dprb_attn_bwd(_ptr(qkv), _ptr(attn_mask), _ptr(ctx), _ptr(lse), _ptr(dctx), _ptr(dqkv),
                                    _ptr(dbias), nseq, S, heads, float(dropout_p), int(site_seed), _stream()),
          "dprb_attn_bwd")
    return dqkv


def attn_cls_fwd(qkv, attn_mask, nseq, S, heads, dropout_p=0.0, site_seed=0):
    """Single-query attention of the pruned last layer (test hook): (ctx_cls bf16 [nseq, H], probs fp32 [nseq, heads, S])."""
    H = heads * 64
    ctx = torch.empty(nseq, H, dtype=torch.bfloat16, device=qkv.device)
    probs = torch.empty(nseq, heads, S, dtype=torch.float32, device=qkv.device)
    check(_lib.load().dprb_attn_cls_fwd(_ptr(qkv), _ptr(attn_mask), _ptr(ctx), _ptr(probs), nseq, S, heads,
                                        float(dropout_p), int(site_seed), _stream()), "dprb_attn_cls_fwd")
    return ctx, probs


def attn_cls_bwd(qkv, probs, dctx_cls, nseq, S, heads, dropout_p=0.0, site_seed=0, dqkv=None):
    """dqkv bf16 [nseq*S, 3H], every element written (dqkv: optional preallocated output)."""
    if dqkv is None:
        dqkv = torch.empty_like(qkv)
    check(_lib.load().dprb_attn_cls_bwd(_ptr(qkv), _ptr(probs), _ptr(dctx_cls), _ptr(dqkv), nseq, S, heads,
                                        float(dropout_p), int(site_seed), _stream()), "dprb_attn_cls_bwd")
    return dqkv


class ScoreCtx:
    """What the tensor-core scoring forward leaves for its backward: the workspace holding the bf16 operand splits
    (and room for the recomputed W tiles), plus the masks / labels / lse the recomputation needs."""

    __slots__ = ("ws", "col_mask", "pair_mask", "labels", "lse", "shape", "local")

    def __init__(self, ws, col_mask, pair_mask, labels, lse, shape, local):
        self.ws, self.col_mask, self.pair_mask, self.labels, self.lse = ws, col_mask, pair_mask, labels, lse
        self.shape, self.local = shape, local


def _round_up8(d):
    return (d + 7) // 8 * 8


def score_fwd(q, c, col_mask, labels, inv_temperature, want_logits=False, pair_mask=None, local=None):
    """Fused scoring + CE forward.  Returns (loss_sum[1], lse[Q], logits or None, ctx): `ctx` (ScoreCtx) is what
    score_bwd needs.  local = (nq, nc) sizes backward's W tiles.  The kernels take d % 8 == 0; other widths are
    zero-padded, which adds exactly 0 to every dot product."""
    Q, d = q.shape
    C = c.shape[0]
    d8 = _round_up8(d)
    if d8 != d:
        q = torch.nn.functional.pad(q, (0, d8 - d))
        c = torch.nn.functional.pad(c, (0, d8 - d))
    lib = _lib.load()
    lse = torch.empty(Q, dtype=torch.float32, device=q.device)
    loss_sum = torch.zeros(1, dtype=torch.float32, device=q.device)
    nq, nc = local if local is not None else (0, 0)
    nbytes = lib.dprb_score_tc_workspace_bytes(Q, C, d8, nq, nc)
    ws = torch.empty(int(nbytes) + 256, dtype=torch.uint8, device=q.device)
    off = (-ws.data_ptr()) % 256
    logits = torch.empty(Q, C, dtype=torch.float32, device=q.device) if want_logits else None
    check(lib.dprb_score_tc_fwd(_ptr(q), _ptr(c), _ptr(col_mask), _ptr(pair_mask), _ptr(labels), float(inv_temperature),
                                _ptr(lse), _ptr(loss_sum), _ptr(logits), Q, C, d8, nq, nc, ws.data_ptr() + off,
                                ws.numel() - off, _stream()), "dprb_score_tc_fwd")
    return loss_sum, lse, logits, ScoreCtx(ws, col_mask, pair_mask, labels, lse, (Q, C, d), (nq, nc))


def score_bwd(ctx, grad_scale, inv_temperature, q0, nq, c0, nc):
    """dq[nq, d], dc[nc, d] of mean-over-Q CE for the rank-local rows / columns; tiles are recomputed (ScoreCtx)."""
    Q, C, d = ctx.shape
    d8 = _round_up8(d)
    assert (nq, nc) == tuple(ctx.local), "score_fwd must be told the local (nq, nc) that backward asks for"
    dq = torch.empty(nq, d8, dtype=torch.float32, device=ctx.ws.device)
    dc = torch.empty(nc, d8, dtype=torch.float32, device=ctx.ws.device)
    off = (-ctx.ws.data_ptr()) % 256
    check(_lib.load().dprb_score_tc_bwd(_ptr(ctx.col_mask), _ptr(ctx.pair_mask), _ptr(ctx.labels), _ptr(ctx.lse),
                                        float(grad_scale), float(inv_temperature), _ptr(dq), _ptr(dc), Q, C, d8, q0,
                                        nq, c0, nc, ctx.ws.data_ptr() + off, ctx.ws.numel() - off, _stream()),
          "dprb_score_tc_bwd")
    return dq[:, :d], dc[:, :d]


_SQERR_WS = {}


def sqerr(x, t, want_dx=True):
    """Squared-error sum (include/dprb.h dprb_sqerr_fwd): x, t fp32 [rows, d] with unit column stride.  Returns
    (loss_sum fp32 [1], dx = 2 (x - t) fp32 [rows, d] or None)."""
    if x.dim() != 2 or x.shape != t.shape:
        raise ValueError(f"squared error needs two [rows, d] operands of one shape (got {tuple(x.shape)} and "
                         f"{tuple(t.shape)})")
    if x.dtype != torch.float32 or t.dtype != torch.float32:
        raise ValueError(f"squared error needs fp32 operands (got {x.dtype} and {t.dtype})")
    x = x if x.stride(1) == 1 else x.contiguous()
    t = t if t.stride(1) == 1 else t.contiguous()
    rows, d = x.shape
    lib = _lib.load()
    loss_sum = torch.empty(1, dtype=torch.float32, device=x.device)
    dx = torch.empty(rows, d, dtype=torch.float32, device=x.device) if want_dx else None
    nbytes = int(lib.dprb_sqerr_workspace_bytes(rows, d))
    buf = _SQERR_WS.get(x.device)
    if buf is None or buf.numel() < nbytes:
        buf = _SQERR_WS[x.device] = torch.empty(max(nbytes, 8), dtype=torch.uint8, device=x.device)
    check(lib.dprb_sqerr_fwd(_ptr(x), max(x.stride(0), d), _ptr(t), max(t.stride(0), d), rows, d, _ptr(loss_sum),
                             _ptr(dx), d, buf.data_ptr(), buf.numel(), _stream()), "dprb_sqerr_fwd")
    return loss_sum, dx


def sumsq(g, out):
    check(_lib.load().dprb_sumsq_f32(_ptr(g), g.numel(), _ptr(out), _stream()), "dprb_sumsq_f32")
    return out


def adamw_step(p, g, m, v, shadow, lr, beta1, beta2, eps, weight_decay, step, grad_scale=1.0, sumsq_buf=None,
               max_norm=0.0):
    check(_lib.load().dprb_adamw_step(_ptr(p), _ptr(g), _ptr(m), _ptr(v), _ptr(shadow), p.numel(), float(lr),
                                      float(beta1), float(beta2), float(eps), float(weight_decay), int(step),
                                      float(grad_scale), _ptr(sumsq_buf), float(max_norm), _stream()),
          "dprb_adamw_step")


LAMB_CHUNK = 8192  # elements per partial sum of the LAMB norms (32 KiB of fp32); a multiple of 4


class LambPlan:
    """Device-side chunk plan + workspace of dprb_lamb_step for one arena cut into contiguous segments of `seg_sizes`
    elements (one per parameter tensor).  Built once per layout; chunks never straddle a segment."""

    def __init__(self, seg_sizes, device, chunk=LAMB_CHUNK):
        sizes = np.asarray(list(seg_sizes), dtype=np.int64)
        if sizes.ndim != 1 or sizes.size == 0 or (sizes <= 0).any() or (sizes % 4).any() or chunk % 4:
            raise ValueError("LambPlan: segments must be non-empty and multiples of 4 elements")
        per = (sizes + chunk - 1) // chunk
        seg_chunk = np.concatenate([[0], np.cumsum(per)])
        chunk_seg = np.repeat(np.arange(sizes.size, dtype=np.int64), per)
        seg_start = np.concatenate([[0], np.cumsum(sizes)])
        within = np.arange(int(seg_chunk[-1]), dtype=np.int64) - seg_chunk[chunk_seg]
        chunk_off = np.append(seg_start[chunk_seg] + within * chunk, seg_start[-1])
        self.numel = int(seg_start[-1])
        self.nchunks, self.nseg = int(seg_chunk[-1]), int(sizes.size)
        self.plan = torch.from_numpy(np.concatenate([chunk_off, chunk_seg, seg_chunk])).to(device)
        nbytes = int(_lib.load().dprb_lamb_workspace_bytes(self.nchunks, self.nseg))
        self.workspace = torch.empty(nbytes, dtype=torch.uint8, device=device)

    def trust_scale(self):
        """step_size * trust ratio per segment as written by the last dprb_lamb_step with this plan."""
        return self.workspace[:4 * (2 * self.nchunks + self.nseg)].view(torch.float32)[2 * self.nchunks:]


def lamb_step(p, g, m, v, shadow, plan, lr, beta1, beta2, eps, weight_decay, clamp_value, adam, debias, step,
              grad_scale=1.0, sumsq_buf=None, max_norm=0.0):
    if p.numel() != plan.numel:
        raise ValueError(f"lamb_step: arena has {p.numel()} elements, the plan covers {plan.numel}")
    check(_lib.load().dprb_lamb_step(_ptr(p), _ptr(g), _ptr(m), _ptr(v), _ptr(shadow), p.numel(), _ptr(plan.plan),
                                     plan.nchunks, plan.nseg, float(lr), float(beta1), float(beta2), float(eps),
                                     float(weight_decay), float(clamp_value), int(bool(adam)), int(bool(debias)),
                                     int(step), float(grad_scale), _ptr(sumsq_buf), float(max_norm),
                                     _ptr(plan.workspace), plan.workspace.numel(), _stream()),
          "dprb_lamb_step")


def madgrad_step(p, g, grad_sum_sq, s, x0, shadow, lr, momentum, weight_decay, eps, k, grad_scale=1.0, sumsq_buf=None,
                 max_norm=0.0):
    check(_lib.load().dprb_madgrad_step(_ptr(p), _ptr(g), _ptr(grad_sum_sq), _ptr(s), _ptr(x0), _ptr(shadow),
                                        p.numel(), float(lr), float(momentum), float(weight_decay), float(eps), int(k),
                                        float(grad_scale), _ptr(sumsq_buf), float(max_norm), _stream()),
          "dprb_madgrad_step")


def cast_f32_bf16(src, dst):
    check(_lib.load().dprb_cast_f32_bf16(_ptr(src), _ptr(dst), src.numel(), _stream()), "dprb_cast_f32_bf16")
    return dst


def cast_bf16_f32(src, dst):
    check(_lib.load().dprb_cast_bf16_f32(_ptr(src), _ptr(dst), src.numel(), _stream()), "dprb_cast_bf16_f32")
    return dst


SEQCLS_MAX_LABELS = 16   # include/dprb.h DPRB_SEQCLS_MAX_LABELS


def seqcls_head_fwd(pre, weight, bias=None):
    """Cross-encoder classification head after its dense layer: pre fp32 [N, H], weight fp32 [L, H], bias fp32 [L]
    -> (logits fp32 [N, L] = tanh(pre) @ weight.T + bias, score fp32 [N] = max over labels)."""
    N, H = pre.shape
    L = weight.shape[0]
    logits = torch.empty(N, L, dtype=torch.float32, device=pre.device)
    score = torch.empty(N, dtype=torch.float32, device=pre.device)
    check(_lib.load().dprb_seqcls_head_fwd(_ptr(pre), _ptr(weight), _ptr(bias), _ptr(logits), _ptr(score), N, H, L,
                                           _stream()), "dprb_seqcls_head_fwd")
    return logits, score


SEQCLS_GROUP_MAX = 64    # include/dprb.h DPRB_SEQCLS_GROUP_MAX
DROP_SITE_HEAD, DROP_SITE_HEAD_IN = 4, 5   # dropout sites (layer 0) of the cross-encoder head (include/dprb.h)
_GROUP_CE_WS = {}


def seqcls_group_ce_check(rows, H, G):
    """The limits of dprb_seqcls_group_ce on the host (ValueError, no device needed); returns the number of groups."""
    if not 2 <= G <= SEQCLS_GROUP_MAX:
        raise ValueError(f"grouped cross-entropy needs 2 <= group size <= {SEQCLS_GROUP_MAX} (got {G})")
    if rows <= 0 or rows % G:
        raise ValueError(f"{rows} rows do not form whole groups of {G}")
    if H % 8 or not 0 < H <= 1024:
        raise ValueError(f"grouped cross-entropy needs a hidden size that is a multiple of 8 and <= 1024 (got {H})")
    return rows // G


def seqcls_group_ce(pre, weight, bias, labels, G, dropout_p=0.0, dropout_seed=0):
    """Grouped softmax cross-entropy of a one-label head and its backward (include/dprb.h dprb_seqcls_group_ce):
    pre fp32 [B*G, H], weight fp32 [1, H], bias fp32 [1] or None, labels int64 [B].  Returns (loss fp32 [1] = mean over
    groups, logits fp32 [B*G], dpre bf16 [B*G, H], dweight fp32 [1, H], dbias fp32 [1]), the gradients of that loss."""
    N, H = pre.shape
    B = seqcls_group_ce_check(N, H, G)
    if weight.shape != (1, H):
        raise ValueError(f"grouped cross-entropy trains one label: weight must be [1, {H}] (got {tuple(weight.shape)})")
    if labels.shape != (B,):
        raise ValueError(f"labels must be [{B}] (got {tuple(labels.shape)})")
    dev = pre.device
    lib = _lib.load()
    loss = torch.empty(1, dtype=torch.float32, device=dev)
    logits = torch.empty(N, dtype=torch.float32, device=dev)
    dpre = torch.empty(N, H, dtype=torch.bfloat16, device=dev)
    dweight = torch.empty(1, H, dtype=torch.float32, device=dev)
    dbias = torch.empty(1, dtype=torch.float32, device=dev)
    nbytes = int(lib.dprb_seqcls_group_ce_workspace_bytes(B, H))
    buf = _GROUP_CE_WS.get(dev)
    if buf is None or buf.numel() < nbytes:
        buf = _GROUP_CE_WS[dev] = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    labels = labels.to(dev, torch.int64).contiguous()
    check(lib.dprb_seqcls_group_ce(_ptr(pre.contiguous()), _ptr(weight.contiguous()), _ptr(bias), _ptr(labels), B, G, H,
                                   float(dropout_p), int(dropout_seed) & 0xFFFFFFFFFFFFFFFF, _ptr(loss), _ptr(logits),
                                   _ptr(dpre), _ptr(dweight), _ptr(dbias), buf.data_ptr(), buf.numel(), _stream()),
          "dprb_seqcls_group_ce")
    return loss, logits, dpre, dweight, dbias


_SEARCH_WS = {}


def _search_ws(nbytes, device):
    """Caller-owned workspace, cached per device and grown on demand (queues are reused across calls)."""
    buf = _SEARCH_WS.get(device)
    if buf is None or buf.numel() < nbytes:
        buf = torch.empty(int(nbytes), dtype=torch.uint8, device=device)
        _SEARCH_WS[device] = buf
    return buf


def search_topk(queries, corpus, k, index_offset=0, reference_ranking=False):
    """Fused inner-product search + top-k: queries [Q, d], corpus [N, d] (both fp16 or both bf16, contiguous)
    -> (scores fp32 [Q, k] descending, row ids int64 [Q, k]); never materialises the [Q, N] score matrix.
    reference_ranking: order by the fp16-rounded score, as the reference's topk over its fp16 einsum does."""
    assert queries.dtype == corpus.dtype and queries.dtype in (torch.float16, torch.bfloat16)
    assert queries.is_contiguous() and corpus.is_contiguous() and queries.shape[1] == corpus.shape[1]
    lib = _lib.load()
    Q, d = queries.shape
    N = corpus.shape[0]
    nbytes = lib.dprb_search_workspace_bytes(Q, int(k))
    if nbytes < 0:
        check(1, "dprb_search_workspace_bytes")
    ws = _search_ws(nbytes, queries.device)
    scores = torch.empty(Q, k, dtype=torch.float32, device=queries.device)
    index = torch.empty(Q, k, dtype=torch.int64, device=queries.device)
    check(lib.dprb_search_topk(_ptr(queries), _ptr(corpus),
                               (1 if queries.dtype == torch.bfloat16 else 0) | (0x100 if reference_ranking else 0), Q, N, d,
                               int(k), int(index_offset), _ptr(scores), _ptr(index), _ptr(ws), ws.numel(),
                               _stream()), "dprb_search_topk")
    return scores, index


def topk_merge(scores, index, k):
    """k best of each row of scores [Q, total] fp32 with their index [Q, total] int64 entries (shard merge)."""
    assert scores.dtype == torch.float32 and index.dtype == torch.int64 and scores.shape == index.shape
    assert scores.is_contiguous() and index.is_contiguous()
    lib = _lib.load()
    Q, total = scores.shape
    ws = torch.empty(int(lib.dprb_topk_merge_workspace_bytes(Q, total)), dtype=torch.uint8, device=scores.device)
    out_s = torch.empty(Q, k, dtype=torch.float32, device=scores.device)
    out_i = torch.empty(Q, k, dtype=torch.int64, device=scores.device)
    check(lib.dprb_topk_merge(_ptr(scores), _ptr(index), Q, total, int(k), _ptr(out_s), _ptr(out_i), _ptr(ws),
                              ws.numel(), _stream()), "dprb_topk_merge")
    return out_s, out_i


def encoder_fwd_tokens(w, b, out):
    """Token-level encoder forward: every token of the last layer, bf16 [nseq*S, H] written into `out` (contiguous
    CUDA).  w / b: the dprb_encoder_weights / dprb_encoder_batch structs (b.save_for_backward must be 0)."""
    check(_lib.load().dprb_encoder_fwd_tokens(ctypes.byref(w), ctypes.byref(b), _ptr(out), _stream()),
          "dprb_encoder_fwd_tokens")
    return out


MAXSIM_POOLS = {"sum": 0, "max": 1}   # include/dprb.h DPRB_MAXSIM_SUM / DPRB_MAXSIM_MAX
MAXSIM_MAX_S, MAXSIM_MAX_P = 512, 1024


def maxsim_check(SQ, SD, P):
    """ValueError for the shapes dprb_maxsim_fwd refuses (token 0 of each side is skipped)."""
    if P % 8 or not 8 <= P <= MAXSIM_MAX_P:
        raise ValueError(f"MaxSim needs the token dimension to be a multiple of 8 and at most {MAXSIM_MAX_P} (got {P})")
    for name, S in (("query", SQ), ("passage", SD)):
        if not 2 <= S <= MAXSIM_MAX_S:
            raise ValueError(f"MaxSim needs {name} sequences of 2 .. {MAXSIM_MAX_S} tokens (got {S})")


def maxsim(q, d, q_mask, d_mask, q_index, pool="sum"):
    """ColBERT MaxSim scores of pairs: q bf16 [nq, SQ, P] (projected query tokens), d bf16 [B, SD, P] (passage tokens),
    int masks [nq, SQ] / [B, SD] (None: every token real), q_index [B] (the query row of each pair; a CPU tensor is
    range-checked without a device sync) -> score fp32 [B] = sum (or max) over query tokens 1.. of the max over passage
    tokens 1.. of q . d, masked tokens counting as zero vectors (include/dprb.h dprb_maxsim_fwd)."""
    if pool not in MAXSIM_POOLS:
        raise ValueError(f"MaxSim pool must be one of {sorted(MAXSIM_POOLS)} (got {pool!r})")
    if q.dim() != 3 or d.dim() != 3 or q.shape[2] != d.shape[2]:
        raise ValueError(f"MaxSim needs q [nq, SQ, P] and d [B, SD, P] (got {tuple(q.shape)} and {tuple(d.shape)})")
    nq, SQ, P = q.shape
    B, SD, _ = d.shape
    maxsim_check(SQ, SD, P)
    q_index = torch.as_tensor(q_index)
    if q_index.shape != (B,):
        raise ValueError(f"MaxSim needs one query index per pair ({B}), got shape {tuple(q_index.shape)}")
    if B and (int(q_index.min()) < 0 or int(q_index.max()) >= nq):
        raise ValueError(f"MaxSim query indices must lie in [0, {nq})")
    assert q.dtype == d.dtype == torch.bfloat16 and q.is_contiguous() and d.is_contiguous()
    dev = d.device
    idx = q_index.to(dev, torch.int32).contiguous()
    qm = None if q_mask is None else q_mask.to(dev, torch.int32).contiguous()
    dm = None if d_mask is None else d_mask.to(dev, torch.int32).contiguous()
    score = torch.empty(B, dtype=torch.float32, device=dev)
    check(_lib.load().dprb_maxsim_fwd(_ptr(q), _ptr(d), _ptr(qm), _ptr(dm), _ptr(idx), nq, SQ, B, SD, P,
                                      MAXSIM_POOLS[pool], _ptr(score), _stream()), "dprb_maxsim_fwd")
    return score


MAXSIM_MAX_EXPERTS = 8   # include/dprb.h dprb_maxsim_expert_fwd: 1 <= KQ, KD <= 8


def maxsim_expert_check(SQ, SD, P, KQ, KD, Pc=None):
    """ValueError for the shapes dprb_maxsim_expert_fwd refuses (Pc: the CLS width, None without a CLS term)."""
    maxsim_check(SQ, SD, P)
    for name, K in (("query", KQ), ("passage", KD)):
        if not 1 <= K <= MAXSIM_MAX_EXPERTS:
            raise ValueError(f"expert MaxSim needs 1 .. {MAXSIM_MAX_EXPERTS} experts per {name} token (got {K})")
    if Pc is not None and (Pc % 8 or not 8 <= Pc <= MAXSIM_MAX_P):
        raise ValueError(f"expert MaxSim needs the CLS dimension to be a multiple of 8 and at most {MAXSIM_MAX_P} "
                         f"(got {Pc})")


def maxsim_expert(q, d, q_ids, q_w, d_ids, d_w, q_index, pool="sum", q_cls=None, d_cls=None):
    """COIL / CITADEL scores of pairs (include/dprb.h dprb_maxsim_expert_fwd): q bf16 [nq, SQ, P], d bf16 [B, SD, P]
    (unmasked tokens, token 0 included), expert ids [nq, SQ, KQ] / [B, SD, KD] (int) and weights (fp32, 0 on masked
    tokens) of the same shape, q_index [B] (a CPU tensor is range-checked without a device sync), optional CLS vectors
    bf16 [nq, Pc] / [B, Pc] -> score fp32 [B] = sum (or max) over query rows (i, a) of the max over passage columns
    (j, b) of q_i . d_j * wq[i, a] * wd[j, b] where the ids agree and 0 where they differ, plus q_cls . d_cls."""
    if pool not in MAXSIM_POOLS:
        raise ValueError(f"MaxSim pool must be one of {sorted(MAXSIM_POOLS)} (got {pool!r})")
    if q.dim() != 3 or d.dim() != 3 or q.shape[2] != d.shape[2]:
        raise ValueError(f"MaxSim needs q [nq, SQ, P] and d [B, SD, P] (got {tuple(q.shape)} and {tuple(d.shape)})")
    nq, SQ, P = q.shape
    B, SD, _ = d.shape
    if q_ids.dim() != 3 or q_ids.shape[:2] != (nq, SQ) or q_w.shape != q_ids.shape:
        raise ValueError(f"expert MaxSim needs query ids and weights [{nq}, {SQ}, KQ] (got {tuple(q_ids.shape)} and "
                         f"{tuple(q_w.shape)})")
    if d_ids.dim() != 3 or d_ids.shape[:2] != (B, SD) or d_w.shape != d_ids.shape:
        raise ValueError(f"expert MaxSim needs passage ids and weights [{B}, {SD}, KD] (got {tuple(d_ids.shape)} and "
                         f"{tuple(d_w.shape)})")
    if (q_cls is None) != (d_cls is None):
        raise ValueError("expert MaxSim needs both CLS operands or neither")
    Pc = None
    if q_cls is not None:
        Pc = q_cls.shape[-1]
        if q_cls.shape != (nq, Pc) or d_cls.shape != (B, Pc):
            raise ValueError(f"expert MaxSim needs CLS vectors [{nq}, Pc] and [{B}, Pc] (got {tuple(q_cls.shape)} and "
                             f"{tuple(d_cls.shape)})")
    maxsim_expert_check(SQ, SD, P, q_ids.shape[2], d_ids.shape[2], Pc)
    q_index = torch.as_tensor(q_index)
    if q_index.shape != (B,):
        raise ValueError(f"MaxSim needs one query index per pair ({B}), got shape {tuple(q_index.shape)}")
    if B and (int(q_index.min()) < 0 or int(q_index.max()) >= nq):
        raise ValueError(f"MaxSim query indices must lie in [0, {nq})")
    assert q.dtype == d.dtype == torch.bfloat16 and q.is_contiguous() and d.is_contiguous()
    if q_cls is not None:
        assert q_cls.dtype == d_cls.dtype == torch.bfloat16 and q_cls.is_contiguous() and d_cls.is_contiguous()
    dev = d.device
    idx = q_index.to(dev, torch.int32).contiguous()
    qi, qw = q_ids.to(dev, torch.int32).contiguous(), q_w.to(dev, torch.float32).contiguous()
    di, dw = d_ids.to(dev, torch.int32).contiguous(), d_w.to(dev, torch.float32).contiguous()
    score = torch.empty(B, dtype=torch.float32, device=dev)
    check(_lib.load().dprb_maxsim_expert_fwd(_ptr(q), _ptr(d), _ptr(qi), _ptr(qw), _ptr(di), _ptr(dw), _ptr(q_cls),
                                             _ptr(d_cls), _ptr(idx), nq, SQ, B, SD, P, qi.shape[2], di.shape[2],
                                             0 if Pc is None else Pc, MAXSIM_POOLS[pool], _ptr(score), _stream()),
          "dprb_maxsim_expert_fwd")
    return score


SPLADE_MAX_K = 1024   # include/dprb.h dprb_splade_pool_fwd: K % 8 == 0, 8 <= K <= 1024


def splade_pool_check(N, V, K, ldx=None, ldw=None, ldo=None, T=0):
    """ValueError for the shapes dprb_splade_pool_fwd refuses (ldx / ldw default to K, ldo to V)."""
    ldx, ldw, ldo = K if ldx is None else ldx, K if ldw is None else ldw, V if ldo is None else ldo
    if K % 8 or not 8 <= K <= SPLADE_MAX_K:
        raise ValueError(f"SPLADE pool needs the hidden width K to be a multiple of 8 in 8 .. {SPLADE_MAX_K} (got {K})")
    for name, ld in (("ldx", ldx), ("ldw", ldw)):
        if ld % 8 or ld < K:
            raise ValueError(f"SPLADE pool needs {name} to be a multiple of 8 and at least K={K} (got {ld})")
    if V < 1 or N < 1:
        raise ValueError(f"SPLADE pool needs V >= 1 and N >= 1 (got V={V}, N={N})")
    if ldo < V:
        raise ValueError(f"SPLADE pool needs ldo >= V={V} (got {ldo})")
    if not 0 <= T < 0x7FFFFF00:
        raise ValueError(f"SPLADE pool needs 0 <= T < 2^31 rows (got {T})")


def splade_pool(x, W, off, K, bias=None, out=None):
    """SPLADE max-pool of compacted tokens (include/dprb.h dprb_splade_pool_fwd): x fp16 [T, ldx] (the tokens' head
    transforms, rows of sequence n at off[n] .. off[n+1] - 1), W fp16 [V, ldw] (the decoder rows), off int [N + 1]
    (non-decreasing), bias fp32 [V] or None; only the first K columns of x and W are read -> fp32 [N, V] =
    log1p(relu(max over each sequence's rows of x . W + bias)), 0 for an empty sequence.  `out` may be a preallocated
    fp32 [N, ldo] tensor with unit column stride (ldo >= V)."""
    if x.dim() != 2 or W.dim() != 2 or x.dtype != torch.float16 or W.dtype != torch.float16:
        raise ValueError("SPLADE pool needs fp16 x [T, ldx] and W [V, ldw]")
    if x.stride(1) != 1 or W.stride(1) != 1:
        raise ValueError("SPLADE pool needs x and W with unit column stride")
    T, V = x.shape[0], W.shape[0]
    off = torch.as_tensor(off)
    N = off.numel() - 1
    if x.shape[1] < K or W.shape[1] < K:
        raise ValueError(f"SPLADE pool reads K={K} columns of x {tuple(x.shape)} and W {tuple(W.shape)}")
    ldo = V if out is None else out.stride(0)
    splade_pool_check(N, V, K, x.stride(0), W.stride(0), ldo, T)
    dev = W.device
    off = off.to(dev, torch.int32).contiguous()
    if out is None:
        out = torch.empty(N, V, dtype=torch.float32, device=dev)
    assert out.dtype == torch.float32 and out.shape[0] >= N and out.shape[1] >= V and out.stride(1) == 1
    b = None if bias is None else bias.to(dev, torch.float32).contiguous()
    check(_lib.load().dprb_splade_pool_fwd(_ptr(x) if T else None, x.stride(0), _ptr(W), W.stride(0), _ptr(b),
                                           _ptr(off), T, N, V, int(K), _ptr(out), ldo, _stream()),
          "dprb_splade_pool_fwd")
    return out


EXPERT_GROUP_CONTEXT_ID, EXPERT_GROUP_PER_SEQUENCE = 1, 2   # include/dprb.h DPRB_EXPERT_GROUP_*
EXPERT_GROUP_MAX_V = 1 << 24


def expert_group_check(N, S, K, P, V, context_id=False):
    """ValueError for the shapes dprb_expert_group refuses (P is not read in context-id mode)."""
    if N < 1 or not 2 <= S <= MAXSIM_MAX_S:
        raise ValueError(f"expert grouping needs N >= 1 sequences of 2 .. {MAXSIM_MAX_S} tokens (got N={N}, S={S})")
    if not 1 <= K <= MAXSIM_MAX_EXPERTS:
        raise ValueError(f"expert grouping needs 1 .. {MAXSIM_MAX_EXPERTS} experts per token (got {K})")
    if N * S * K >= 1 << 31:
        raise ValueError(f"expert grouping needs N*S*K < 2^31 entries (got {N * S * K})")
    if not 1 <= V < EXPERT_GROUP_MAX_V:
        raise ValueError(f"expert grouping needs a vocabulary of 1 .. 2^24 - 1 experts (got {V})")
    if not context_id and (P % 8 or not 8 <= P <= MAXSIM_MAX_P):
        raise ValueError(f"expert grouping needs the token dimension to be a multiple of 8 and at most {MAXSIM_MAX_P} "
                         f"(got {P})")


_GROUP_WS = {}


def expert_group(reps, ids, w, mask, V, threshold=0.0, tokens=None, per_sequence=False):
    """Kept (token, expert) entries of one encoded batch grouped by expert (include/dprb.h dprb_expert_group).

    reps bf16 [N, S, P] (unit column stride, token 0 included; None in context-id mode), ids [N, S, K] (int, in
    [0, V)), w fp32 [N, S, K], mask [N, S]; entry (n, s, k) is kept when s >= 1, mask != 0 and w > threshold.  With
    ``tokens`` [N, S] (context-id mode) the weight test is skipped and the payload is the token id.  Entries are sorted
    by expert id (``per_sequence``: by (n, expert id)), ties in (n, s, k) order.

    Returns device tensors of the E kept entries: (expert int32 [E], seq int32 [E], token int32 [E], weight fp32 [E],
    payload fp32 [E, P] = weight * float(rep), or fp32 [E] = float(token id)).  Reading E is the call's one host
    synchronisation."""
    if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (reps, w)):
        raise ValueError("expert grouping runs forward only: call it under torch.no_grad()")
    if ids.dim() != 3 or w.shape != ids.shape or mask.shape != ids.shape[:2]:
        raise ValueError(f"expert grouping needs ids and weights [N, S, K] and a mask [N, S] (got {tuple(ids.shape)}, "
                         f"{tuple(w.shape)} and {tuple(mask.shape)})")
    N, S, K = ids.shape
    ctx = tokens is not None
    if ctx:
        if tuple(tokens.shape) != (N, S):
            raise ValueError(f"expert grouping needs token ids [{N}, {S}] (got {tuple(tokens.shape)})")
        P = 0
    else:
        if reps is None or reps.dim() != 3 or reps.shape[:2] != (N, S):
            raise ValueError(f"expert grouping needs reps [{N}, {S}, P] (got "
                             f"{None if reps is None else tuple(reps.shape)})")
        P = reps.shape[2]
    expert_group_check(N, S, K, P, V, ctx)
    dev = ids.device
    lib = _lib.load()
    ids32 = ids.to(dev, torch.int32).contiguous()
    w32 = w.to(dev, torch.float32).contiguous()
    m32 = mask.to(dev, torch.int32).contiguous()
    tok32 = tokens.to(dev, torch.int32).contiguous() if ctx else None
    if not ctx:
        assert reps.dtype == torch.bfloat16 and reps.stride(2) == 1 and reps.stride(0) == S * reps.stride(1)
    cap = max(N * (S - 1) * K, 1)
    count = torch.empty(1, dtype=torch.int32, device=dev)
    expert, seq, tok = (torch.empty(cap, dtype=torch.int32, device=dev) for _ in range(3))
    weight = torch.empty(cap, dtype=torch.float32, device=dev)
    payload = torch.empty((cap,) if ctx else (cap, P), dtype=torch.float32, device=dev)
    nbytes = int(lib.dprb_expert_group_workspace_bytes(N, S, K))
    buf = _GROUP_WS.get(dev)
    if buf is None or buf.numel() < nbytes + 256:
        buf = _GROUP_WS[dev] = torch.empty(nbytes + 256, dtype=torch.uint8, device=dev)
    off = (-buf.data_ptr()) % 256
    flags = (EXPERT_GROUP_CONTEXT_ID if ctx else 0) | (EXPERT_GROUP_PER_SEQUENCE if per_sequence else 0)
    check(lib.dprb_expert_group(_ptr(ids32), _ptr(w32), _ptr(m32), _ptr(tok32), None if ctx else _ptr(reps),
                                0 if ctx else reps.stride(1), N, S, K, P, int(V), float(threshold), flags,
                                _ptr(count), _ptr(expert), _ptr(seq), _ptr(tok), _ptr(weight), _ptr(payload),
                                buf.data_ptr() + off, buf.numel() - off, _stream()), "dprb_expert_group")
    E = int(count.item())
    return expert[:E], seq[:E], tok[:E], weight[:E], payload[:E]


EXPERT_SEARCH_MAX_P = 1024        # include/dprb.h dprb_expert_search: P, Pc multiples of 8, 8 .. 1024
EXPERT_SEARCH_MAX_K = 1024
EXPERT_SEARCH_GROUP = 64          # query rows per work group (the kernel's wgmma M)
EXPERT_SEARCH_CLS_TILE = 128      # CLS rows per CLS tile (the kernel's wgmma N)
EXPERT_SEARCH_TILE_WINDOW = 112   # an index tile holds the runs that start in one 112-entry window of its expert
EXPERT_SEARCH_TERM_LIMIT = 2.0 ** 30   # bound on a query's sum of |terms| (int64 fixed point at 2^-32)
FP16_MAX = 65504.0


def expert_search_check(P, Pc, V, E, N, k):
    """ValueError for the shapes dprb_expert_search refuses (Pc None: no CLS term)."""
    for name, w in (("payload", P), ("CLS", Pc)):
        if w is not None and (w % 8 or not 8 <= w <= EXPERT_SEARCH_MAX_P):
            raise ValueError(f"expert search needs the {name} width to be a multiple of 8 in 8 .. "
                             f"{EXPERT_SEARCH_MAX_P} (got {w})")
    if not 1 <= V < EXPERT_GROUP_MAX_V:
        raise ValueError(f"expert search needs a vocabulary of 1 .. 2^24 - 1 experts (got {V})")
    if not 0 <= E < 1 << 31:
        raise ValueError(f"expert search needs fewer than 2^31 index entries (got {E})")
    if not 1 <= N < 1 << 31:
        raise ValueError(f"expert search needs 1 .. 2^31 - 1 passages (got {N})")
    if not 1 <= k <= min(EXPERT_SEARCH_MAX_K, N):
        raise ValueError(f"expert search needs 1 <= topk <= min({EXPERT_SEARCH_MAX_K}, passages={N}) (got {k})")


def expert_search_block_queries(N):
    """Queries per search block: the [Qb, N] int64 accumulator stays within the library's fixed 2 GiB budget."""
    return int(_lib.load().dprb_expert_search_block_queries(int(N)))


def expert_search_tiles(expert, row, V, window=EXPERT_SEARCH_TILE_WINDOW):
    """Index tiles of entries sorted by (expert, row) (host int arrays [E]): (tile_bounds int32 [T + 1], tile_ptr int64
    [V + 1] = each expert's first tile).  A tile is the runs (one row's entries of one expert) that start in the same
    ``window``-entry window of their expert, so no run is split and a run longer than a tile stays whole."""
    expert = np.asarray(expert, dtype=np.int64)
    row = np.asarray(row, dtype=np.int64)
    E = expert.size
    if E == 0:
        return np.zeros(1, np.int32), np.zeros(V + 1, np.int64)
    ptr = np.zeros(V + 1, np.int64)
    np.cumsum(np.bincount(expert, minlength=V), out=ptr[1:])
    rs = np.flatnonzero(np.r_[True, (expert[1:] != expert[:-1]) | (row[1:] != row[:-1])])
    ex = expert[rs]
    win = (rs - ptr[ex]) // window
    starts = rs[np.r_[True, (ex[1:] != ex[:-1]) | (win[1:] != win[:-1])]]
    tile_ptr = np.zeros(V + 1, np.int64)
    np.cumsum(np.bincount(expert[starts], minlength=V), out=tile_ptr[1:])
    return np.r_[starts, E].astype(np.int32), tile_ptr


def expert_search_groups(q_expert, tile_ptr, n_cls, N):
    """Work groups of one query block: query entries sorted by expert (host int [Eq]) cut into runs of <= 64 of one
    expert, each with its expert's tiles (experts without postings are dropped), then ``n_cls`` queries' CLS rows in
    groups of 64 with the ceil(N / 128) CLS tiles.  Returns (groups int32 [G, 4], item_end int32 [G], items)."""
    q_expert = np.asarray(q_expert, dtype=np.int64)
    V = tile_ptr.size - 1
    parts = []
    if q_expert.size:
        starts = np.flatnonzero(np.r_[True, q_expert[1:] != q_expert[:-1]])
        counts = np.diff(np.r_[starts, q_expert.size])
        xs = q_expert[starts]
        known = xs < V
        ntiles = np.zeros(xs.size, np.int64)
        ntiles[known] = tile_ptr[xs[known] + 1] - tile_ptr[xs[known]]
        ng = (counts + EXPERT_SEARCH_GROUP - 1) // EXPERT_SEARCH_GROUP
        gi = np.repeat(np.arange(xs.size), ng)
        j = np.arange(gi.size) - np.repeat(np.cumsum(ng) - ng, ng)
        lo = starts[gi] + EXPERT_SEARCH_GROUP * j
        rows = np.minimum(EXPERT_SEARCH_GROUP, counts[gi] - EXPERT_SEARCH_GROUP * j)
        first = np.where(known[gi], tile_ptr[np.minimum(xs[gi], V - 1)], 0)
        g = np.stack([np.zeros_like(lo), lo, rows, first, ntiles[gi]], 1)
        parts.append(g[g[:, 4] > 0])
    if n_cls:
        lo = np.arange(0, n_cls, EXPERT_SEARCH_GROUP)
        rows = np.minimum(EXPERT_SEARCH_GROUP, n_cls - lo)
        nt = (N + EXPERT_SEARCH_CLS_TILE - 1) // EXPERT_SEARCH_CLS_TILE
        parts.append(np.stack([np.ones_like(lo), lo, rows, np.zeros_like(lo), np.full_like(lo, nt)], 1))
    g = np.concatenate(parts) if parts else np.zeros((0, 5), np.int64)
    end = np.cumsum(g[:, 4])
    items = int(end[-1]) if end.size else 0
    if items >= 1 << 31:
        raise ValueError(f"expert search block has {items} work items (2^31 or more): search fewer queries at once")
    return np.ascontiguousarray(g[:, :4], dtype=np.int32), end.astype(np.int32), items


_EXPERT_SEARCH_WS = {}


def expert_search(payload, row, tile_bounds, P, cls, row_ids, q_payload, q_seq, q_cls, Qb, groups, item_end, items,
                  k):
    """One query block through dprb_expert_search (include/dprb.h).  Index: payload fp16 [E, ldp], row int32 [E],
    tile_bounds int32 [T + 1], cls fp16 [N, ldc] or None, row_ids int64 [N] (the corpus id of each row).  Queries:
    q_payload fp16 [Eq, ldp] sorted by expert, q_seq int32 [Eq] in [0, Qb), q_cls fp16 [Qb, ldc] or None; groups /
    item_end / items from expert_search_groups (device int32).  Returns (scores fp32 [Qb, k], ids int64 [Qb, k])."""
    lib = _lib.load()
    dev = row_ids.device
    N = row_ids.numel()
    E, Eq = row.numel(), q_seq.numel()
    for t in (payload, q_payload) + ((cls, q_cls) if cls is not None else ()):
        assert t.dtype == torch.float16 and t.is_contiguous() and t.device == dev
    assert q_payload.shape[1] == payload.shape[1]
    Pc = 0 if cls is None else int(cls.shape[1])
    if cls is not None:
        assert q_cls is not None and q_cls.shape == (Qb, cls.shape[1])
    nbytes = int(lib.dprb_expert_search_workspace_bytes(N, int(Qb)))
    buf = _EXPERT_SEARCH_WS.get(dev)
    if buf is None or buf.numel() < nbytes + 256:
        _EXPERT_SEARCH_WS[dev] = None                          # free the old buffer before taking the new one
        buf = _EXPERT_SEARCH_WS[dev] = torch.empty(nbytes + 256, dtype=torch.uint8, device=dev)
    off = (-buf.data_ptr()) % 256
    scores = torch.empty(Qb, k, dtype=torch.float32, device=dev)
    ids = torch.empty(Qb, k, dtype=torch.int64, device=dev)
    check(lib.dprb_expert_search(_ptr(payload), _ptr(row), _ptr(tile_bounds), E, tile_bounds.numel() - 1, int(P),
                                 payload.shape[1], _ptr(cls), Pc, 0 if cls is None else cls.shape[1], _ptr(row_ids), N,
                                 _ptr(q_payload), _ptr(q_seq), Eq, _ptr(q_cls), int(Qb), _ptr(groups), _ptr(item_end),
                                 groups.shape[0], int(items), int(k), _ptr(scores), _ptr(ids), buf.data_ptr() + off,
                                 buf.numel() - off, _stream()), "dprb_expert_search")
    return scores, ids


SPARSE_SEARCH_TILE = 2048         # include/dprb.h DPRB_SPARSE_SEARCH_TILE: postings per work item
SPARSE_SEARCH_MAX_K = 1024


def sparse_search_check(V, nnz, N, k):
    """ValueError for the shapes dprb_sparse_search refuses (host-only: needs no GPU)."""
    if not 1 <= V < 1 << 31:
        raise ValueError(f"sparse search needs a vocabulary of 1 .. 2^31 - 1 terms (got {V})")
    if not 0 <= nnz < 1 << 40:
        raise ValueError(f"sparse search needs fewer than 2^40 postings (got {nnz})")
    if not 1 <= N < 1 << 31:
        raise ValueError(f"sparse search needs 1 .. 2^31 - 1 passages (got {N})")
    if not 1 <= k <= min(SPARSE_SEARCH_MAX_K, N):
        raise ValueError(f"sparse search needs 1 <= topk <= min({SPARSE_SEARCH_MAX_K}, passages={N}) (got {k})")


def sparse_search_block_queries(N):
    """Queries per search block: the [Qb, N] int64 accumulator stays within the library's fixed 2 GiB budget."""
    return int(_lib.load().dprb_sparse_search_block_queries(int(N)))


def sparse_search_items(term_ptr, q_term):
    """Work items of one query block: term_ptr host int64 [V + 1], q_term host int [Eq] -> (item_end int32 [Eq], items),
    each entry owning ceil(postings of its term / SPARSE_SEARCH_TILE) items."""
    q_term = np.asarray(q_term, dtype=np.int64)
    n = term_ptr[q_term + 1] - term_ptr[q_term]
    end = np.cumsum((n + SPARSE_SEARCH_TILE - 1) // SPARSE_SEARCH_TILE)
    items = int(end[-1]) if end.size else 0
    if items >= 1 << 31:
        raise ValueError(f"sparse search block has {items} work items (2^31 or more): search fewer queries at once")
    return end.astype(np.int32), items


_SPARSE_SEARCH_WS = {}


def sparse_search(row, weight, term_ptr, nnz, row_ids, q_term, q_weight, q_seq, Qb, item_end, items, k):
    """One query block through dprb_sparse_search (include/dprb.h).  Index: row int32 / weight fp16 [>= nnz rounded up
    to 8], term_ptr int64 [V + 1], row_ids int64 [N] (the id returned for each row).  Queries: q_term int32 [Eq] in
    [0, V), q_weight fp32 [Eq], q_seq int32 [Eq] in [0, Qb), item_end int32 [Eq] / items from sparse_search_items
    (all device tensors).  Returns (scores fp32 [Qb, k], ids int64 [Qb, k])."""
    lib = _lib.load()
    dev = row_ids.device
    N, V, Eq = row_ids.numel(), term_ptr.numel() - 1, q_term.numel()
    assert row.dtype == torch.int32 and weight.dtype == torch.float16 and term_ptr.dtype == torch.int64
    assert row.numel() >= (nnz + 7) // 8 * 8 and weight.numel() >= (nnz + 7) // 8 * 8
    assert q_term.dtype == torch.int32 and q_weight.dtype == torch.float32 and q_seq.dtype == torch.int32
    assert item_end.dtype == torch.int32 and item_end.numel() == Eq and q_weight.numel() == Eq == q_seq.numel()
    for t in (row, weight, term_ptr, row_ids, q_term, q_weight, q_seq, item_end):
        assert t.is_contiguous() and t.device == dev
    nbytes = int(lib.dprb_sparse_search_workspace_bytes(N, int(Qb)))
    buf = _SPARSE_SEARCH_WS.get(dev)
    if buf is None or buf.numel() < nbytes + 256:
        _SPARSE_SEARCH_WS[dev] = None                          # free the old buffer before taking the new one
        buf = _SPARSE_SEARCH_WS[dev] = torch.empty(nbytes + 256, dtype=torch.uint8, device=dev)
    off = (-buf.data_ptr()) % 256
    scores = torch.empty(Qb, k, dtype=torch.float32, device=dev)
    ids = torch.empty(Qb, k, dtype=torch.int64, device=dev)
    check(lib.dprb_sparse_search(_ptr(row), _ptr(weight), _ptr(term_ptr), int(nnz), int(V), _ptr(row_ids), N,
                                 _ptr(q_term), _ptr(q_weight), _ptr(q_seq), _ptr(item_end), int(Eq), int(items),
                                 int(Qb), int(k), _ptr(scores), _ptr(ids), buf.data_ptr() + off, buf.numel() - off,
                                 _stream()), "dprb_sparse_search")
    return scores, ids
