#!/usr/bin/env python
"""FILM harness: BASELINE.json configs[2] / SURVEY.md section 8d config 3 - FILM VFI, 4x multiplier, synthetic 1080p
clip, frame pairs sharded over the GPUs of one box with an NCCL gather of the output frames.

    python tools/bench_film.py [--frames 9] [--multiplier 4] [--steps 3] [--warmup 3] [--pairs 4] [--layers] [--no-cpu]
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P \
        tools/bench_film.py --frames 17 ...

(bench.py stays the driver's contract for the RIFE north-star metric; this is the same contract for the FILM config.)
One step = the FILM node over this rank's `--frames`-frame clip (weak scaling: every rank has its own clip of the same
shape): (frames-1) x (multiplier-1) interpolated frames, each one `Interpolator.forward` on a pair; `--pairs` pairs that
are at the same step of their bisection schedules go through one library call.
  value        : interpolated frames/s, clip resident in HBM, CUDA events, max over ranks; N > 1: each rank's output
                 frames are gathered on rank 0 over NCCL inside the step
  e2e          : the same through `FILM_VFI.vfi` with host frames (pinned), H2D and D2H inside the timed region
  roofline     : tensor-core TFLOP/s of the whole forward (MACs of the unpadded channels, counted by the library)
                 against the measured bf16 peak; --layers adds per-layer times of every streamconv launch
  cpu_baseline : oracle/film.py (== the reference's PyTorch-CPU path) on ONE 1080p pair (rank 0, N = 1)
Inputs are larger than L2 (25 MB per frame, ~6 GB of workspace traffic per forward).
"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=9, help="source frames per GPU")
    ap.add_argument("--multiplier", type=int, default=4)
    ap.add_argument("--pairs", type=int, default=4, help="pairs per library call (film_node.PAIRS_PER_PASS)")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--h", type=int, default=1080)
    ap.add_argument("--w", type=int, default=1920)
    ap.add_argument("--layers", action="store_true")
    ap.add_argument("--no-cpu", action="store_true")
    a = ap.parse_args()
    a.warmup = max(a.warmup, 3)

    import __graft_entry__ as ge
    ge.load_package()
    import bench as B                     # ClockSampler, _peaks
    import cfi_b200.film_node as FN
    from cfi_b200.engine import FilmEngine
    from oracle import film as OF         # synthetic weights / clips; the CPU baseline leg

    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    torch.cuda.set_device(local_rank)
    dist = None
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))

    def barrier():
        if dist is not None:
            dist.barrier()
        torch.cuda.synchronize()

    H, W, nf, m = a.h, a.w, a.frames, a.multiplier
    FN.PAIRS_PER_PASS = a.pairs
    sd = OF.synthetic_state_dict(0)
    eng = FilmEngine(sd, device=local_rank, dtype="float32")
    clip = OF.synthetic_clip(nf, H, W, seed=1234 + rank)
    n_out = (nf - 1) * m + 1
    n_interp = (nf - 1) * (m - 1)
    order = FN.inference_order(m - 1)
    gathered = [torch.empty((n_out - 1, H, W, 3), dtype=torch.float32, device="cuda") for _ in range(world)] \
        if (dist is not None and rank == 0) else None

    # ---- device-resident: the node's schedule on device tensors (what film_node.FILM_VFI.vfi does between its copies)
    dev_clip = clip.cuda()
    dev_out = torch.empty((n_out - 1, H, W, 3), dtype=torch.float32, device="cuda")  # without the closing frame

    def step_device():
        for c0 in range(0, nf - 1, a.pairs):
            chunk = list(range(c0, min(c0 + a.pairs, nf - 1)))
            nc = len(chunk)
            store = torch.empty((nc, m + 1, H, W, 3), dtype=torch.float32, device="cuda")
            for j, i in enumerate(chunk):
                store[j, 0].copy_(dev_clip[i])
                store[j, m].copy_(dev_clip[i + 1])
            flat = store.view(nc * (m + 1), H, W, 3)
            for lo, hi, new in order:
                mid = eng.forward(flat, [j * (m + 1) + lo for j in range(nc)], [j * (m + 1) + hi for j in range(nc)], clamp=True)
                store[:, new].copy_(mid)
            for j, i in enumerate(chunk):
                dev_out[i * m:(i + 1) * m].copy_(store[j, :m])
        if dist is not None:
            dist.gather(dev_out, gathered, dst=0)

    for _ in range(a.warmup):
        step_device()
    barrier()
    sampler = B.ClockSampler(local_rank)
    if rank == 0:
        sampler.start()
        sampler.wait_first()
    barrier()
    l0 = eng.launch_count()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t_begin = time.time()
    e0.record()
    for _ in range(a.steps):
        step_device()
    e1.record()
    barrier()
    t_end = time.time()
    ms_dev = e0.elapsed_time(e1)
    launches = eng.launch_count() - l0
    last_b = ((nf - 1) % a.pairs) or min(a.pairs, nf - 1)   # pairs in the last library call of a step
    macs_per_call = eng.last_macs() / last_b
    clocks = sampler.stop(t_begin, t_end) if rank == 0 else None

    # ---- end to end through the node (host frames in, host frames out)
    host_in = clip.contiguous().pin_memory()
    node = FN.FILM_VFI()
    out = None
    for _ in range(2):
        (out,) = node.vfi("film_net_fp32.pt", host_in, multiplier=m, _engine=eng)
    barrier()
    t0 = time.perf_counter()
    for _ in range(a.steps):
        (out,) = node.vfi("film_net_fp32.pt", host_in, multiplier=m, _engine=eng)
    barrier()
    sec_e2e = time.perf_counter() - t0
    same = bool(torch.equal(out[1:m], dev_out[1:m].cpu()))  # host path == device path on the first pair's new frames

    tt = torch.tensor([ms_dev, sec_e2e * 1e3], dtype=torch.float64, device="cuda")
    if dist is not None:
        dist.all_reduce(tt, op=dist.ReduceOp.MAX)
    ms_dev, ms_e2e = tt.tolist()

    if rank == 0:
        peaks = B._peaks()
        total = n_interp * world
        value = total * a.steps / (ms_dev / 1e3)
        tf = 2.0 * macs_per_call * value / world / 1e12   # per GPU: the peak is one GPU's
        line = {
            "metric": "interpolated frames/sec @1080p FILM %dx" % m if (H, W) == (1080, 1920) else
                      "interpolated frames/sec @%dx%d FILM %dx" % (W, H, m),
            "value": value, "unit": "frames/s", "n_gpus": world, "steps": a.steps, "warmup": a.warmup,
            "ms_per_step": ms_dev / a.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "f16", "dtype_note": "conv operands fp16, fp32 accumulate (registers); images, flows, warps' weights fp32",
            "data": "synthetic",
            "config": {"workload": f"FILM VFI, {m}x multiplier, {nf}-frame synthetic {H}x{W} clip per GPU "
                                   f"(BASELINE configs[2] shape; {nf - 1} pairs x {m - 1} forward calls)",
                       "pairs_per_call": a.pairs,
                       "parallelism": f"frame-pair shards x{world}, output frames gathered on rank 0 by NCCL" if world > 1 else "1 GPU",
                       "weights": "seeded synthetic (oracle.film.synthetic_state_dict(0)); no checkpoint ships",
                       "l2": "inputs larger than L2"},
            "e2e": {"value": total * a.steps / (ms_e2e / 1e3), "unit": "frames/s", "ms_per_step": ms_e2e / a.steps,
                    "h2d_bytes_per_step": nf * H * W * 3 * 4, "d2h_bytes_per_step": n_out * H * W * 3 * 4,
                    "host_equals_device_path": same},
            "gpu_launches": launches, "clocks": clocks,
            "roofline": {"bound": "tensor", "kernel": "whole Interpolator.forward (streamconv + HBM kernels)",
                         "achieved": tf, "peak": peaks["tflops_sustained"] or peaks["tflops"], "unit": "TFLOP/s",
                         "frac": tf / (peaks["tflops_sustained"] or peaks["tflops"]), "traffic": None,
                         "peak_source": peaks["source"] + ", sustained figure (inside a long step)",
                         "gmacs_per_call": macs_per_call / 1e9},
        }
        if a.layers:
            rows = []
            lvl = [(H >> l, W >> l) for l in range(7)]
            todo = [(0, 2 * j + k, j, f"extract.{j}.{k}") for j in range(4) for k in (0, 1) if not (j == 0 and k == 0)]
            todo += [(1, 4 * p + c, p, f"flow.{'shared' if p == 3 else p}.{c}") for p in range(4) for c in range(4)]
            todo += [(2, 3 * k + c, 3 - k, f"fuse.{k}.{c}") for k in range(4) for c in range(3)]
            flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
            for g, layer, l, label in todo:
                plan = eng.layer_plan(g, layer)
                hh, ww = lvl[l]
                x0 = torch.zeros((1, hh, ww, plan["c0"]), dtype=torch.float16, device="cuda")
                x1 = torch.zeros((1, hh, ww, plan["c1"]), dtype=torch.float16, device="cuda") if plan["c1"] else None
                y = torch.empty((1, hh, ww, plan["n_total"]), dtype=torch.float16, device="cuda")
                ts = []
                for i in range(8):
                    flush.zero_()
                    e0.record()
                    eng.debug_conv(g, layer, x0, x1, y, 1, hh, ww)
                    e1.record()
                    torch.cuda.synchronize()
                    if i >= 3:
                        ts.append(e0.elapsed_time(e1))
                us = sum(ts) / len(ts) * 1e3
                fl = 2.0 * plan["ksize"] ** 2 * (plan["c0"] + plan["c1"]) * plan["n_total"] * hh * ww
                rows.append(dict(layer=label, level=l, us=round(us, 1), tflops_padded=round(fl / us / 1e6, 1), **plan))
            line["layers"] = rows
        if world == 1 and not a.no_cpu:
            torch.set_num_threads(min(32, os.cpu_count() or 1))
            x = clip[:2].permute(0, 3, 1, 2)
            t0 = time.perf_counter()
            OF.interpolator_forward(sd, x[0:1], x[1:2], torch.full((1, 1), 0.5))
            sec = time.perf_counter() - t0
            line["cpu_baseline"] = {"value": 1.0 / sec, "unit": "frames/s", "cores": torch.get_num_threads(), "kind": "port",
                                    "sample": f"one {H}x{W} pair = one forward call ({sec:.1f} s), oracle/film.py == the "
                                              "reference's PyTorch-CPU path"}
        print(json.dumps(line))
    eng.close()
    if dist is not None:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
