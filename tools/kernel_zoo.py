#!/usr/bin/env python3
"""One launch of every hot kernel at BASELINE config 2's context-encoder shapes (T = 131 072 tokens, BERT-base) and the
config-3 scoring shape, for `ncu --set full` (one capture per kernel family):

  ncu --set full --clock-control none -o gpurun_out/zoo python tools/kernel_zoo.py          # ~45 launches

Order = the order of the printed index, so a launch in the report can be mapped to its role.
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from dpr_scale_b200 import ops

T, H, I, S, HEADS = 131072, 768, 3072, 128, 12
dev, bf = "cuda", torch.bfloat16
g = torch.Generator(device=dev).manual_seed(0)
rnd = lambda *s, dt=bf, sc=1.0: (torch.randn(*s, device=dev, generator=g) * sc).to(dt)
idx = []


def gemm(name, M, N, K, a_mn, b_mn, epi, aux=None, out2=False, colsum=False, f32=False, flags=0, out_dt=bf, p=0.0):
    A = rnd(K, M) if a_mn else rnd(M, K)
    B = rnd(K, N, sc=0.02) if b_mn else rnd(N, K, sc=0.02)
    D = torch.zeros(M, N, device=dev, dtype=torch.float32 if f32 else out_dt)
    bias = torch.zeros(N, device=dev) if (epi in (0, 1, 2) and not f32) else None
    o2 = torch.empty(M, N, device=dev, dtype=bf) if out2 else None
    cs = torch.zeros(N, device=dev) if colsum else None
    ops.gemm(A, B, D, M, N, K, M if a_mn else K, N if b_mn else K, N, a_mn, b_mn, epi | flags, bias, aux,
             N if aux is not None else 0, o2, 1.0, 0 if f32 else 1, cs, p, 12345)
    idx.append(name)


x16 = rnd(T, H, dt=torch.float16)
gemm("gemm fwd QKV (bias)", T, 3 * H, H, 0, 0, 0)
gemm("gemm fwd attn-out (bias + dropout + fp16 residual -> fp16 sum)", T, H, H, 0, 0, 2, aux=x16,
     flags=ops.GEMM_AUX_F16 | ops.GEMM_OUT_F16, out_dt=torch.float16, p=0.1)
gemm("gemm fwd FFN-in (bias + GELU, gelu' saved)", T, I, H, 0, 0, 1, out2=True)
gemm("gemm fwd FFN-out (bias + dropout + fp16 residual -> fp16 sum)", T, H, I, 0, 0, 2, aux=x16,
     flags=ops.GEMM_AUX_F16 | ops.GEMM_OUT_F16, out_dt=torch.float16, p=0.1)
gemm("gemm dgrad W2 (dGELU + colsum)", T, I, H, 0, 1, 3, aux=rnd(T, I), colsum=True)
gemm("gemm dgrad W1 (+ residual grad)", T, H, I, 0, 1, 2, aux=rnd(T, H))
gemm("gemm dgrad Wo", T, H, H, 0, 1, 0)
gemm("gemm dgrad Wqkv (+ residual grad)", T, H, 3 * H, 0, 1, 2, aux=rnd(T, H))
gemm("gemm wgrad W2 (split-K fp32 atomics)", H, I, T, 1, 1, 4, f32=True)
gemm("gemm wgrad W1", I, H, T, 1, 1, 4, f32=True)
gemm("gemm wgrad Wo", H, H, T, 1, 1, 4, f32=True)
gemm("gemm wgrad Wqkv", 3 * H, H, T, 1, 1, 4, f32=True)

qkv = rnd(T, 3 * H)
seed = ops.dropout_site_seed(7, 3, 1)
ctx, lse = ops.attn_fwd(qkv, None, T // S, S, HEADS, True, 0.1, seed); idx.append("attention fwd (wgmma, dropout 0.1)")
dctx = rnd(T, H)
ops.attn_bwd(qkv, None, ctx, lse, dctx, T // S, S, HEADS, torch.zeros(3 * H, device=dev), 0.1, seed); idx.append("attention bwd (wgmma, dropout 0.1)")

z16 = rnd(T, H, dt=torch.float16, sc=2.0)
gamma, beta = torch.ones(H, device=dev), torch.zeros(H, device=dev)
yres = torch.empty(T, H, dtype=torch.float16, device=dev)
y, stats, _ = ops.ln_fwd(z16, gamma, beta, 1e-12, 0, yres); idx.append("LayerNorm fwd (fp16 sum in, bf16 + fp16 out)")
dg, db, dbias = (torch.zeros(H, device=dev) for _ in range(3))
ops.ln_bwd(rnd(T, H), z16, stats, gamma, dg, db, dbias, None, 1, 0.1, seed); idx.append("LayerNorm bwd (dense, + dropout-masked copy, dgamma/dbeta/dbias)")

V, P = 30522, 512
word, pos, typ = rnd(V, H, dt=torch.float32, sc=0.02), rnd(P, H, dt=torch.float32, sc=0.02), rnd(2, H, dt=torch.float32, sc=0.02)
ids = torch.randint(1000, 30000, (T,), device=dev, generator=g)
tts = torch.zeros(T, dtype=torch.long, device=dev)
pids = (torch.arange(T, device=dev) % S)
y0, st0 = ops.embed_ln_fwd(ids, tts, pids, word, pos, typ, gamma, beta, 1e-12, 0.1, 7, yres); idx.append("embedding gather + LayerNorm fwd")
dword, dpos, dtyp = torch.zeros_like(word), torch.zeros_like(pos), torch.zeros_like(typ)
ops.embed_ln_bwd(rnd(T, H), ids, tts, pids, word, pos, typ, gamma, st0, dword, dpos, dtyp, dg, db, 0.1, 7); idx.append("embedding LayerNorm bwd + scatter-add")

n = 108_891_648
p_, g_, m_, v_ = (torch.randn(n, device=dev) for _ in range(4))
v_.abs_()
sh = torch.empty(n, dtype=bf, device=dev)
ss = torch.zeros(1, device=dev)
ops.sumsq(g_, ss); idx.append("gradient sum of squares (clip)")
ops.adamw_step(p_, g_, m_, v_, sh, 1e-5, 0.9, 0.999, 1e-8, 0.0, 1, 1.0, ss, 2.0); idx.append("fused clip + AdamW + bf16 shadow refresh")
del p_, g_, m_, v_, sh

Q, C, d = 1024, 8192, 768
q, c = torch.randn(Q, d, device=dev, generator=g), torch.randn(C, d, device=dev, generator=g)
mask = torch.zeros(C, dtype=torch.uint8, device=dev)
labels = torch.randint(0, C, (Q,), device=dev, generator=g)
_, _, _, sctx = ops.score_fwd(q, c, mask, labels, 1.0, False, None, (128, 1024))
idx += ["score: bf16 split of q", "score: bf16 split of c", "score fwd (wgmma tiles + online softmax + NLL), 1024 x 8192 x 768"]
ops.score_bwd(sctx, 1.0, 1.0, 256, 128, 2048, 1024)
idx += ["score bwd: W tiles recomputed (local rows + local columns)"] + ["score bwd GEMM %d/6" % i for i in range(1, 7)]
torch.cuda.synchronize()
for i, nm in enumerate(idx):
    print(i, nm)
