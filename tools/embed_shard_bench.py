#!/usr/bin/env python3
"""configs[4] of BASELINE.json - the generate_embeddings.py path, sharded over N GPUs - measured through the repo's own
task class:

  python tools/embed_shard_bench.py --passages-per-rank 500000 --batch 128 --out /tmp/emb            # 1 GPU
  python -m torch.distributed.run --nproc-per-node 8 ... tools/embed_shard_bench.py ...              # 8 GPUs

Every rank drives ``GenerateEmbeddingsTask.test_step`` (dpr_scale_b200/task/dpr_eval_task.py, the drop-in for
/root/reference/dpr_scale/task/dpr_eval_task.py:13-49) over its contiguous shard of a synthetic, pre-tokenised corpus
(BERT-base, S = 128, all sequences full length - the named shape): pinned host batches -> H2D -> forward-only encoder ->
async D2H into the pinned ring -> rows appended to ``reps_{rank:04}.pkl`` by the streaming writer; then the barrier of
:49.  The path shards with NO collective (utils/utils.py:83-91), so N GPUs are N independent streams.

One JSON line (rank 0): passages/s of the whole job = total passages / max over ranks of the device-timed region
(CUDA events around the loop + the final drain), per-rank numbers, the model-FLOP rate (22.35 GFLOP per passage forward) against the measured dense bf16 peak, bytes moved per passage, the size of the files written, peak host RSS
(the reference holds the shard twice in RAM: 2 x 4 x 768 x passages bytes).
"""
import argparse
import json
import os
import resource
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist

BERT_BASE = dict(model_type="bert", vocab_size=30522, hidden_size=768, num_hidden_layers=12, num_attention_heads=12,
                 intermediate_size=3072, max_position_embeddings=512, type_vocab_size=2, layer_norm_eps=1e-12,
                 pad_token_id=0)
FWD_FLOP_PER_TOKEN = 174_587_904          # BERT-base S = 128: 2 x (4H^2 + 2HI) + 4SH per layer x 12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passages-per-rank", type=int, default=200_000)
    ap.add_argument("--batch", type=int, default=128, help="conf/datamodule/generate.yaml:5 test_batch_size")
    ap.add_argument("--seq", type=int, default=128)
    ap.add_argument("--out", default="/tmp/dprb_embed_bench")
    ap.add_argument("--keep", action="store_true", help="keep the reps_*.pkl files")
    ap.add_argument("--distinct-batches", type=int, default=64, help="pinned synthetic batches cycled through")
    args = ap.parse_args()
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        from dpr_scale_b200.utils.dist_init import init_process_group
        init_process_group(dev)
    from dpr_scale_b200.task.dpr_eval_task import GenerateEmbeddingsTask
    task = GenerateEmbeddingsTask(ctx_embeddings_dir=args.out, checkpoint_path="", transform={}, datamodule=None,
                                  optim={}, shared_model=False,
                                  model={"_target_": "dpr_scale_b200.models.hf_model.HFEncoder.from_config",
                                         "config": BERT_BASE, "dropout": 0.1})
    task.trainer = None
    task.setup("test")
    task = task.to(dev).eval()
    B, S = args.batch, args.seq
    g = torch.Generator().manual_seed(1234 + rank)
    pool = []
    for _ in range(args.distinct_batches):
        ids = torch.randint(1000, 30000, (B, S), generator=g)
        ids[:, 0], ids[:, -1] = 101, 102
        pool.append({"input_ids": ids.pin_memory(), "token_type_ids": torch.zeros(B, S, dtype=torch.long).pin_memory(),
                     "attention_mask": torch.ones(B, S, dtype=torch.long).pin_memory()})
    nb = (args.passages_per_rank + B - 1) // B
    rows_last = args.passages_per_rank - (nb - 1) * B

    def batch(i):
        b = pool[i % len(pool)]
        n = rows_last if i == nb - 1 else B
        return {"contexts_ids": {k: v[:n].to(dev, non_blocking=True) for k, v in b.items()}}

    for i in range(5):                                   # warm-up (kernels, allocator, pinned ring), then a fresh file
        task.test_step(batch(0), i)
    task.test_epoch_end([])
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    e0.record()
    for i in range(nb):
        task.test_step(batch(i), i)
    e1.record()
    out_file = task.test_epoch_end([])                   # drains the ring, closes the pickle, barrier (:49)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    dev_s = e0.elapsed_time(e1) / 1e3
    size = os.path.getsize(out_file)
    rss_gb = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2 ** 20
    stats = torch.tensor([dev_s, wall, float(size), rss_gb], dtype=torch.float64, device=dev)
    if world > 1:
        allst = [torch.zeros_like(stats) for _ in range(world)]
        dist.all_gather(allst, stats)
    else:
        allst = [stats]
    if rank == 0:
        import pickle
        with open(out_file, "rb") as f:
            t = pickle.load(f)
        ok = tuple(t.shape) == (args.passages_per_rank, 768) and t.dtype == torch.float32 and bool(torch.isfinite(t).all())
        peaks = {}
        p = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")
        if os.path.exists(p):
            peaks = json.load(open(p))
        peak_tf = peaks.get("bf16_tflops_sustained", 989.0)
        slow_wall = max(float(s[1]) for s in allst)
        slow_dev = max(float(s[0]) for s in allst)
        total = args.passages_per_rank * world
        pps = total / slow_wall
        line = {
            "metric": "passages/sec (generate_embeddings, BERT-base, seq128)", "value": pps, "unit": "passages/s",
            "n_gpus": world, "higher_is_better": True, "scaling": "weak", "dtype": "bf16", "data": "synthetic tokens",
            "config": {"workload": f"generate_embeddings bert-base s{S} batch {B}", "passages_per_rank": args.passages_per_rank,
                       "total_passages": total, "collectives": "none on the data path (contiguous shard per rank; final barrier)"},
            "timed_region": "H2D of every batch + forward-only encoder + async D2H + streaming pickle write + drain + barrier; "
                            "wall clock, max over ranks",
            "wall_s_max_rank": slow_wall, "device_loop_s_max_rank": slow_dev,
            "per_rank_passages_per_s": [args.passages_per_rank / float(s[1]) for s in allst],
            "model_tflops": pps * S * FWD_FLOP_PER_TOKEN / 1e12,
            "frac_of_measured_bf16_peak": pps * S * FWD_FLOP_PER_TOKEN / 1e12 / (peak_tf * world),
            "peak_tflops_per_gpu": peak_tf,
            "h2d_bytes_per_passage": 3 * S * 8, "d2h_bytes_per_passage": 768 * 4,
            "file_bytes_per_rank": [int(s[2]) for s in allst], "host_peak_rss_gb_per_rank": [round(float(s[3]), 2) for s in allst],
            "reference_host_copy_gb_per_rank": round(2 * args.passages_per_rank * 768 * 4 / 2 ** 30, 2),
            "file_check": {"rank0_shape_dtype_finite_ok": bool(ok)},
            "projected_21M_passages_s": 21015324 / pps,
        }
        print(json.dumps(line), flush=True)
    if world > 1:
        dist.barrier()
    if not args.keep:
        try:
            os.remove(out_file)
        except OSError:
            pass
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
