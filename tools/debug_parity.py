import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from tests.test_task_gpu import _task, _batch, _grad_report
from tests.util import load_golden, sub, BERT_TINY_CFG, cosine, rel_l2
from oracle import encoder as oenc, task as otask

g = load_golden("golden_1rank.npz")
T = float(g["temperature"])
task = _task(g)
batch = _batch(g)
# --- probe
enc = task.context_encoder
tokens = batch["contexts_ids"]
probe = torch.randn(8, 128, generator=torch.Generator().manual_seed(3))
sd = {k: v.clone().requires_grad_(True) for k, v in sub(g, "sd_c/").items()}
ref_rep = oenc.encode(sd, BERT_TINY_CFG, tokens)
(ref_rep * probe).sum().backward()
enc.zero_grad()
rep = enc(tokens)
(rep * probe.cuda()).sum().backward()
torch.cuda.synchronize()
print("PROBE rep rel", rel_l2(rep.detach().cpu(), ref_rep.detach()))
for k, p in enc.named_parameters():
    r = sd[k].grad
    if r is None: continue
    got = p.grad.detach().cpu()
    print(f"probe {k:60s} cos {cosine(got, r):.5f} rel {rel_l2(got, r):.4f} refnorm {float(r.norm()):.3e} gotnorm {float(got.norm()):.3e}")
# --- full
for e in (task.query_encoder, task.context_encoder):
    e.zero_grad()
q, c = task(batch["query_ids"], batch["contexts_ids"])
qd, cd = q.detach().cpu().requires_grad_(True), c.detach().cpu().requires_grad_(True)
l_or, _ = otask.in_batch_loss(qd, cd, batch["ctx_mask"], batch["pos_ctx_indices"], T)
l_or.backward()
q.retain_grad(); c.retain_grad()
loss = task.training_step(batch, 0)
print("loss", float(loss), float(l_or), float(g["loss"]))
from dpr_scale_b200 import ops
_, _, _, sctx = ops.score_fwd(q.detach(), c.detach(), batch["ctx_mask"].to(torch.uint8).cuda(), batch["pos_ctx_indices"].cuda(), 1.0 / T, False, None, (4, 8))
dq, dc = ops.score_bwd(sctx, 1.0, 1.0 / T, 0, 4, 0, 8)
print("dq vs oracle", cosine(dq.cpu(), qd.grad), rel_l2(dq.cpu(), qd.grad), "dc", cosine(dc.cpu(), cd.grad), rel_l2(dc.cpu(), cd.grad))
loss.backward()
torch.cuda.synchronize()
for name, e in (("q", task.query_encoder), ("c", task.context_encoder)):
    ref = sub(g, f"grad_{name}/")
    for k, p in e.named_parameters():
        if k not in ref: continue
        r = ref[k]; got = p.grad.detach().cpu()
        print(f"full {name} {k:60s} cos {cosine(got, r):.5f} rel {rel_l2(got, r):.4f} refnorm {float(r.norm()):.3e}")
