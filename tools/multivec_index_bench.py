#!/usr/bin/env python3
"""Throughput of COIL / CITADEL expert-index generation at BERT-base dims (CITADEL: token width 32, CLS 128, S = 256,
batches of 128 passages, topk 1 and 2), one JSON line per measurement:

  index   passages/s of one generation step: this repo's encoder (expert_reps) + dprb_expert_group + the copy of the
          grouped entries to the host, against stock HF (BertForMaskedLM in fp32, the reference's CITADEL head math)
          + the reference's per-entry Python loop restated (one .item() per kept entry)
  group   the grouping alone on one batch's encoder outputs: dprb_expert_group against torch.argsort(stable=True) +
          gather of the same entries

  python tools/multivec_index_bench.py --out h100_multivec_index_bench.jsonl

Times are CUDA-event / synchronised host-clock times on the card named in each line, with its power limit.
"""
import argparse
import collections
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from dpr_scale_b200 import ops  # noqa: E402
from tests import multivec_cases  # noqa: E402

N, S = 128, 256


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def tokens(seed, vocab):
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(S // 2, S + 1, (N,), generator=g)
    ids = torch.randint(1000, vocab, (N, S), generator=g)
    ids[:, 0] = 101
    am = (torch.arange(S)[None] < lens[:, None]).long()
    return {"input_ids": (ids * am).cuda(), "token_type_ids": torch.zeros(N, S, dtype=torch.long).cuda(),
            "attention_mask": am.cuda()}


def ours_step(enc, toks, topk):
    with torch.no_grad():
        reps, ids, w, cls = enc.expert_reps(toks, topk=topk, add_cls=True)
        out = ops.expert_group(reps, ids, w, toks["attention_mask"], enc.config["vocab_size"], 0.0)
        host = [t.cpu() for t in out] + [cls.float().cpu()]
    return host


def reference_step(hf, sd, toks, topk):
    """Stock HF forward + the reference's CITADEL head (citadel_model.py) + its per-entry loop."""
    with torch.no_grad():
        o = hf(**toks, output_hidden_states=True, return_dict=True)
        h = o.hidden_states[-1]
        logits = o.logits[:, 1:]
        am = toks["attention_mask"][:, 1:]
        router = torch.log1p(torch.relu(logits)) * am.unsqueeze(-1)
        w, ids = router.topk(topk, dim=-1)
        rep = torch.nn.functional.linear(h[:, 1:], sd["tok_project.0.weight"], sd["tok_project.0.bias"]) * am.unsqueeze(-1)
        cls = torch.nn.functional.linear(h[:, 0], sd["cls_project.0.weight"], sd["cls_project.0.bias"])
        rep, ids, w, am, cls = rep.cpu(), ids.cpu(), w.cpu(), am.cpu(), cls.cpu()
    results = []
    for b in range(N):
        res = collections.defaultdict(list)
        for r, i, ww, a in zip(rep[b], ids[b], w[b], am[b]):
            if a > 0:
                for x, wx in zip(i, ww):
                    if wx > 0:
                        res[x.item()].append([b, wx, wx * r])
        results.append(res)
    return results


def timed(fn, reps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--ref-steps", type=int, default=2)
    args = ap.parse_args()
    from transformers import BertConfig, BertForMaskedLM
    from dpr_scale_b200.models.citadel_models.citadel_model import CITADELEncoder
    sd, cfg = multivec_cases.bert_base_state_dict("citadel")
    enc = CITADELEncoder.from_config(cfg, *multivec_cases.BASE["citadel"])
    enc.load_state_dict(sd, strict=True)
    enc.cuda()
    hf = BertForMaskedLM(BertConfig(**cfg))
    hf.load_state_dict({k[len("transformer."):]: v for k, v in sd.items() if k.startswith("transformer.")},
                       strict=False)
    hf.cuda().eval()
    sdc = {k: v.cuda() for k, v in sd.items()}
    name = card()
    lines = []
    toks = tokens(0, cfg["vocab_size"])
    for topk in (1, 2):
        ours_step(enc, toks, topk)
        t_ours = timed(lambda: ours_step(enc, toks, topk), args.steps)
        reference_step(hf, sdc, toks, topk)
        t_ref = timed(lambda: reference_step(hf, sdc, toks, topk), args.ref_steps)
        lines.append({"bench": "index", "model": "citadel-bert-base", "topk": topk, "S": S, "batch": N,
                      "ours_passages_per_s": N / t_ours, "reference_passages_per_s": N / t_ref,
                      "speedup": t_ref / t_ours, "gpu": name})
        # the grouping alone on this batch's encoder outputs
        with torch.no_grad():
            reps, ids, w, _ = enc.expert_reps(toks, topk=topk, add_cls=False)
        V, am = cfg["vocab_size"], toks["attention_mask"]
        am32 = am.int()

        def ours_group():
            return ops.expert_group(reps, ids, w, am32, V, 0.0)

        def torch_group():
            keep = (w > 0) & (am32[:, :, None] != 0)
            keep[:, 0] = False
            flat = keep.view(-1).nonzero().squeeze(1)
            x = ids.view(-1)[flat]
            order = torch.argsort(x, stable=True)
            e = flat[order]
            k = ids.shape[2]
            tok = e // k
            pay = w.view(-1)[e][:, None] * reps.view(-1, reps.shape[2])[tok].float()
            return x[order], tok, w.view(-1)[e], pay

        a, b = ours_group(), torch_group()
        assert torch.equal(a[0], b[0].int()) and torch.equal(a[4], b[3])
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        for _ in range(3):
            ours_group(), torch_group()
        ev[0].record()
        for _ in range(args.steps):
            ours_group()
        ev[1].record()
        for _ in range(args.steps):
            torch_group()
        ev[2].record()
        torch.cuda.synchronize()
        lines.append({"bench": "group", "topk": topk, "entries": int(a[0].numel()), "P": int(reps.shape[2]),
                      "ours_ms": ev[0].elapsed_time(ev[1]) / args.steps,
                      "torch_argsort_gather_ms": ev[1].elapsed_time(ev[2]) / args.steps, "gpu": name,
                      "note": "both include their one host sync to size the outputs"})
    for ln in lines:
        print(json.dumps(ln))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for ln in lines:
                f.write(json.dumps(ln) + "\n")


if __name__ == "__main__":
    main()
