"""Speed of one canvas sharded by window across GPUs (parallel.window_shard_plan + the two-phase step + the NCCL exchange) on the 16->128
config in bf16, 128x128 windows, overlap 32, one image per canvas.  One NCCL process per rank, for every rank count in --worlds that the
machine has GPUs for.  Prints one JSON line:
  * per canvas and rank count: ms per canvas step (CUDA events around K steps after warm-up, a barrier on both sides, the maximum over
    ranks; median and min..max over rounds), the share of the step spent from the end of phase (a) to the end of the exchange (the
    transfer plus any wait for a slower neighbour) and in the merge (rank maximum), and the speedup over one rank;
  * on one rank also the one-graph step of the unsharded canvas (super_resolution_windowed's), alternated round by round;
  * the GPU's name, power limit and maximum SM clock, and the SM clock observed right after the timed rounds.

    python tools/gpu_windowed_shard_bench.py [--steps 10] [--warmup 2] [--rounds 3] [--canvases 720x1280,2160x3840] [--worlds 1,2,4,8]
"""
import argparse
import json
import os
import socket
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SCHED = {"schedule": "linear", "n_timestep": 2000, "linear_start": 1e-6, "linear_end": 1e-2}
UNET = dict(in_channel=6, out_channel=3, inner_channel=64, channel_multiplier=[1, 2, 4, 8, 8], attn_res=[16], res_blocks=2, dropout=0.0)
IMAGE, WINDOW, OVERLAP = 128, (128, 128), 32


def smi(fields):
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader"], capture_output=True, text=True)
    return [s.strip() for s in out.stdout.strip().splitlines()[0].split(",")]


def spread(v):
    return {"median_ms_per_step": statistics.median(v), "min": min(v), "max": max(v), "rounds": len(v)}


def worker(rank, world, port, args, path):
    import torch
    import torch.distributed as dist
    import sr3_b200
    from sr3_b200 import parallel
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        torch.manual_seed(0)
        opt = {"phase": "val", "gpu_ids": [0], "distributed": False,
               "model": {"which_model_G": "sr3", "finetune_norm": False, "unet": dict(UNET),
                         "beta_schedule": {"train": dict(SCHED), "val": dict(SCHED)},
                         "diffusion": {"image_size": IMAGE, "channels": 3, "conditional": True}}}
        net = sr3_b200.define_G(opt).to(dev)
        net.set_new_noise_schedule(SCHED, dev)
        net.eval()
        T, K, warm = SCHED["n_timestep"], args.steps, args.warmup
        rows = []
        for H, W in [tuple(int(v) for v in s.split("x")) for s in args.canvases.split(",")]:
            g = torch.Generator().manual_seed(3)
            cond, x_T = (torch.rand(1, 3, H, W, generator=g) * 2 - 1).to(dev), torch.randn(1, 3, H, W, generator=g).to(dev)
            plan = parallel.window_shard_plan(1, H, W, WINDOW, OVERLAP, world)
            sh = plan[rank]
            s = net._windowed_range_sampler(1, H, W, WINDOW, OVERLAP, sh)
            exchange = parallel.p2p_exchange(plan, rank, s.means)
            dist.all_reduce(torch.zeros(1, device=dev))
            whole = net._windowed_sampler(1, H, W, WINDOW, OVERLAP) if world == 1 else None
            step_ms, x_share, m_share, whole_ms = [], [], [], []
            for _ in range(args.rounds):
                s.begin(cond, x_T, 1234, 0)
                s.phase_begin(T - 1)
                for _ in range(warm):
                    s.phase_means(); exchange(); s.phase_merge()
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(3 * K + 1)]
                torch.cuda.synchronize()
                dist.barrier()
                ev[0].record()
                for k in range(K):
                    s.phase_means(); ev[3 * k + 1].record()
                    exchange(); ev[3 * k + 2].record()
                    s.phase_merge(); ev[3 * k + 3].record()
                torch.cuda.synchronize()
                dist.barrier()
                total = ev[0].elapsed_time(ev[3 * K])
                xch = sum(ev[3 * k + 1].elapsed_time(ev[3 * k + 2]) for k in range(K))
                mrg = sum(ev[3 * k + 2].elapsed_time(ev[3 * k + 3]) for k in range(K))
                v = torch.tensor([total / K, xch / total, mrg / total], device=dev, dtype=torch.float64)
                dist.all_reduce(v, op=dist.ReduceOp.MAX)
                step_ms.append(v[0].item()); x_share.append(v[1].item()); m_share.append(v[2].item())
                assert torch.isfinite(s.read_state()[0, :, sh.bands[0][0]:sh.bands[0][1]]).all()
                if whole is not None:                        # the unsharded canvas's one-graph step, alternated with the sharded one
                    whole.begin(cond, x_T, 1234, 0)
                    whole.steps(T - 1, warm)
                    torch.cuda.synchronize()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    whole.steps(T - 1 - warm, K)
                    e1.record()
                    torch.cuda.synchronize()
                    whole_ms.append(e0.elapsed_time(e1) / K)
            row = {"canvas": f"{H}x{W}", "ranks": world, "windows": plan[-1].n1, "windows_per_rank": max(p.n1 - p.n0 for p in plan),
                   "windows_per_pass": s.engine.batch, "received_windows_max": max(sum(m1 - m0 for _, m0, m1 in p.recv) for p in plan),
                   "sharded": spread(step_ms), "exchange_share_median": statistics.median(x_share),
                   "merge_share_median": statistics.median(m_share), "observed_sm_clock": smi("clocks.sm")[0]}
            if whole_ms:
                row["unsharded_one_graph"] = spread(whole_ms)
            rows.append(row)
            del s, whole, exchange
            net._windowed = None
            net.denoise_fn._engines.clear()
            net.denoise_fn._engine_versions.clear()
            torch.cuda.empty_cache()
        if rank == 0:
            with open(path, "w") as fh:
                json.dump(rows, fh)
    finally:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--canvases", default="720x1280,2160x3840")
    ap.add_argument("--worlds", default="1,2,4,8")
    args = ap.parse_args()
    import torch
    import torch.multiprocessing as mp
    assert torch.cuda.is_available(), "this measurement needs an H100"
    n_dev = torch.cuda.device_count()
    name, limit, max_clock = smi("name,power.limit,clocks.max.sm")
    out = {"config": "16->128 (sr_sr3_16_128), bf16, window 128x128, overlap 32, one image per canvas",
           "gpu": {"name": name, "power_limit": limit, "max_sm_clock": max_clock, "devices": n_dev}, "runs": [], "not_measured": []}
    with tempfile.TemporaryDirectory() as tmp:
        for world in [int(w) for w in args.worlds.split(",")]:
            if world > n_dev:
                out["not_measured"].append("%d ranks (%d GPUs visible)" % (world, n_dev))
                continue
            s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
            path = os.path.join(tmp, "w%d.json" % world)
            mp.spawn(worker, args=(world, port, args, path), nprocs=world, join=True)
            with open(path) as fh:
                out["runs"] += json.load(fh)
    one = {r["canvas"]: r["sharded"]["median_ms_per_step"] for r in out["runs"] if r["ranks"] == 1}
    for r in out["runs"]:
        if r["canvas"] in one:
            r["speedup_over_one_rank"] = one[r["canvas"]] / r["sharded"]["median_ms_per_step"]
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
