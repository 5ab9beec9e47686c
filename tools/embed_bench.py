#!/usr/bin/env python3
"""configs[4] (generate_embeddings path): forward-only passage encoding throughput, BERT-base, S = 128.

  python tools/embed_bench.py [batch ...]        default batches: 128 (conf/datamodule/generate.yaml:5) and 1024

Per batch size, one JSON line: passages/s of (a) this repo's encoder in forward-only mode driven like
GenerateEmbeddingsTask (dpr_eval_task.py:32-49: encode, copy to a pinned host buffer asynchronously) with HOST input
batches (pinned -> H2D inside the timed region), (b) the stock HuggingFace BertModel under bf16 autocast on the same
inputs with the reference's per-batch `.cpu()`.  Projects the 21 M-passage corpus on 8 GPUs (the path shards with no
collective: each rank encodes its contiguous slice).
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from dpr_scale_b200.models.hf_model import HFEncoder

CFG = dict(vocab_size=30522, hidden_size=768, num_hidden_layers=12, num_attention_heads=12, intermediate_size=3072,
           max_position_embeddings=512)
FWD_FLOP_PER_TOKEN = 174_587_904          # BERT-base S=128: 2 x (4H^2 + 2HI) + 4SH per layer x 12


def batches(B, S, n, seed=0):
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n):
        ids = torch.randint(1000, 30000, (B, S), generator=g)
        ids[:, 0], ids[:, -1] = 101, 102
        out.append({"input_ids": ids.pin_memory(), "token_type_ids": torch.zeros(B, S, dtype=torch.long).pin_memory(),
                    "attention_mask": torch.ones(B, S, dtype=torch.long).pin_memory()})
    return out


def timed(fn, data, warm=3):
    for b in data[:warm]:
        fn(b)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for b in data[warm:]:
        fn(b)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / (len(data) - warm)


def main():
    dev = torch.device("cuda")
    sizes = [int(x) for x in sys.argv[1:]] or [128, 1024]
    torch.manual_seed(0)
    enc = HFEncoder.from_config(CFG, dropout=0.1).to(dev).eval()
    from transformers import BertConfig, BertModel
    hf = BertModel(BertConfig(**CFG), add_pooling_layer=False).to(dev).eval()
    S = 128
    for B in sizes:
        data = batches(B, S, 3 + max(8, 8192 // B))
        host = [torch.empty(B, 768, dtype=torch.float32).pin_memory() for _ in data]
        it = iter(range(10 ** 9))

        @torch.no_grad()
        def ours(b):
            t = {k: v.to(dev, non_blocking=True) for k, v in b.items()}
            host[next(it) % len(host)].copy_(enc(t), non_blocking=True)

        @torch.no_grad()
        def stock(b):
            t = {k: v.to(dev, non_blocking=True) for k, v in b.items()}
            with torch.autocast("cuda", dtype=torch.bfloat16):
                out = hf(**t)[0][:, 0, :]
            return out.float().cpu()               # dpr_eval_task.py:35: per-batch .cpu()
        ms, ms_stock = timed(ours, data), timed(stock, data)
        pps = B / ms * 1e3
        print(json.dumps({"workload": f"generate_embeddings BERT-base S=128 batch {B}", "passages_per_s": round(pps, 1),
                          "ms_per_batch": round(ms, 3), "tflops": round(pps * S * FWD_FLOP_PER_TOKEN / 1e12, 1),
                          "stock_hf_bf16_passages_per_s": round(B / ms_stock * 1e3, 1),
                          "speedup_vs_stock": round(ms_stock / ms, 2),
                          "h2d_bytes_per_batch": 3 * B * S * 8, "d2h_bytes_per_batch": B * 768 * 4,
                          "projected_21M_passages_8gpu_s": round(21015324 / 8 / pps, 1)}), flush=True)


if __name__ == "__main__":
    main()
