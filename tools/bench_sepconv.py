#!/usr/bin/env python
"""Sepconv harness (BASELINE.json configs[4]: Sepconv VFI 2x, 32-frame 4K clip over 8 GPUs; `bench.py --workload sepconv`).

    python tools/bench_sepconv.py [--frames 5] [--pairs 2] [--steps 5] [--warmup 3] [--h 2160 --w 3840]
    python -m torch.distributed.run --nproc-per-node N ... tools/bench_sepconv.py ...      (one rank per GPU)

Same JSON-line contract as bench.py.  One step = this rank's (frames - 1) frame pairs through `vfi_sepconv_forward`,
`--pairs` pairs per library call (weak scaling: every rank has its own clip shard; for N > 1 the interpolated frames are
gathered on rank 0 by NCCL inside the timed region - the path's only exchange).
  value        : interpolated frames/s, clips resident in HBM, CUDA events, max over ranks
  e2e          : the same through the node call SepconvVFI().vfi(...) on a host tensor (the node's per-pair upload / download
                 loop, vfi_utils.py:149-216, inside the timed region)
  roofline     : the whole Network.forward against the sustained bf16 tensor peak, from the trunk's MACs per pixel
                 (479 KMAC/px, SURVEY.md section 8 row a12); roofline_op: the K = 51 separable-convolution op alone against
                 the fp32 FMA rate (20.8 KMAC/px per frame, two launches)
  cpu_baseline : oracle/sepconv.py (== the reference's PyTorch-CPU path) on one small pair, scaled per pixel
"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

TRUNK_MACS_PER_PX = 479e3   # conv trunk incl. the four 51-channel heads (SURVEY.md section 8 a12, probe)
OP_MACS_PER_PX = 20.8e3     # adaptive separable convolution: 2 frames x 51 x 51 taps x 4 channels (fp32 CUDA cores)
FP32_FMA_TFLOPS = 67.0      # H100 SXM data sheet, FP32 (no measured figure in MEASURED_PEAKS.json)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=5, help="source frames per GPU")
    ap.add_argument("--pairs", type=int, default=2, help="pairs per library call")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--h", type=int, default=2160)
    ap.add_argument("--w", type=int, default=3840)
    ap.add_argument("--no-cpu", action="store_true")
    a = ap.parse_args()
    a.warmup = max(a.warmup, 3)
    import __graft_entry__ as ge
    ge.load_package()
    import bench as B
    from cfi_b200.engine import SepconvEngine
    from cfi_b200 import ops as OPS
    from cfi_b200 import sepconv_node as SN
    from oracle import film as OF      # synthetic clip generator
    from oracle import sepconv as OS   # synthetic weights (no checkpoint ships); the CPU leg

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

    H, W, nf = a.h, a.w, a.frames
    npairs = nf - 1
    sd = OS.synthetic_state_dict(0)
    eng = SepconvEngine(sd, device=local_rank)
    clip = OF.synthetic_clip(nf, H, W, seed=1234 + rank)
    dev_clip = clip.cuda().contiguous()
    out = torch.empty((npairs, H, W, 3), dtype=torch.float32, device="cuda")
    gathered = [torch.empty_like(out) for _ in range(world)] if (dist is not None and rank == 0) else None

    def step_device():
        for lo in range(0, npairs, a.pairs):
            hi = min(lo + a.pairs, npairs)
            eng.forward(dev_clip, list(range(lo, hi)), list(range(lo + 1, hi + 1)), out=out[lo:hi])
        if dist is not None:
            dist.gather(out, gathered, dst=0)

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
    clocks = sampler.stop(t_begin, t_end) if rank == 0 else None
    finite = bool(torch.isfinite(out).all())

    # ---- end to end through the node (host frames in, host frames out; its loop moves one pair at a time)
    node = SN.SepconvVFI()
    res = None
    for _ in range(2):
        (res,) = node.vfi("sepconv.pth", clip, multiplier=2, _engine=eng)
    barrier()
    t0 = time.perf_counter()
    for _ in range(a.steps):
        (res,) = node.vfi("sepconv.pth", clip, multiplier=2, _engine=eng)
    barrier()
    sec_e2e = time.perf_counter() - t0
    same = bool(tuple(res.shape) == (2 * nf - 1, H, W, 3) and torch.equal(res[1], out[0].cpu()))

    tt = torch.tensor([ms_dev, sec_e2e * 1e3], dtype=torch.float64, device="cuda")
    if dist is not None:
        dist.all_reduce(tt, op=dist.ReduceOp.MAX)
    ms_dev, ms_e2e = tt.tolist()

    if rank == 0:
        peaks = B._peaks()
        total = npairs * world
        value = total * a.steps / (ms_dev / 1e3)
        px = float(H * W)
        tf = 2.0 * TRUNK_MACS_PER_PX * px * value / world / 1e12   # per GPU: the peak is one GPU's
        peak_t = peaks["tflops_sustained"] or peaks["tflops"]
        line = {"metric": f"interpolated frames/sec @{W}x{H} Sepconv 2x", "value": value, "unit": "frames/s", "n_gpus": world,
                "steps": a.steps, "warmup": a.warmup, "ms_per_step": ms_dev / a.steps, "higher_is_better": True,
                "scaling": "weak", "vs_baseline": None, "dtype": "f16",
                "dtype_note": "trunk conv operands fp16, fp32 accumulate (registers); the separable-convolution op fp32", "data": "synthetic",
                "config": {"workload": f"Sepconv VFI, 2x multiplier, {nf}-frame synthetic {H}x{W} clip per GPU (BASELINE configs[4] shape)",
                           "pairs_per_call": a.pairs,
                           "parallelism": f"frame-pair shards x{world}, output frames gathered on rank 0 by NCCL" if world > 1 else "1 GPU",
                           "weights": "seeded synthetic (oracle.sepconv.synthetic_state_dict(0)); no checkpoint ships",
                           "l2": "inputs larger than L2"},
                "e2e": {"value": total * a.steps / (ms_e2e / 1e3), "unit": "frames/s", "ms_per_step": ms_e2e / a.steps,
                        "via": "SepconvVFI.vfi (node call; generic_frame_loop moves one pair per call)",
                        "h2d_bytes_per_step": 2 * npairs * H * W * 3 * 4, "d2h_bytes_per_step": npairs * H * W * 3 * 4,
                        "node_output_matches_device_path": same},
                "gpu_launches": launches, "clocks": clocks, "finite": finite,
                "roofline": {"bound": "tensor", "kernel": "whole Network.forward (streamconv EXT trunk + element-wise + K=51 op)",
                             "achieved": tf, "peak": peak_t, "unit": "TFLOP/s", "frac": tf / peak_t, "traffic": None,
                             "peak_source": peaks["source"] + ", sustained figure (inside a long step)",
                             "macs_per_px": TRUNK_MACS_PER_PX}}
        # the op alone, on one frame's shapes (two of these run per interpolated frame)
        he, we = H + H % 2, W + W % 2
        x = torch.rand(1, 4, he + 50, we + 50, device="cuda")
        v = torch.rand(1, 51, he, we, device="cuda")
        hz = torch.rand(1, 51, he, we, device="cuda")
        for _ in range(2):
            OPS.sepconv_func.apply(x, v, hz)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(3):
            OPS.sepconv_func.apply(x, v, hz)
        e1.record()
        torch.cuda.synchronize()
        op_ms = e0.elapsed_time(e1) / 3
        op_tf = 2.0 * (OP_MACS_PER_PX / 2) * he * we / (op_ms * 1e-3) / 1e12
        line["roofline_op"] = {"bound": "fp32 FMA", "kernel": "sepconv_tile_kernel (K = 51, RGB + ones, one frame)", "launch_ms": op_ms,
                               "achieved": op_tf, "peak": FP32_FMA_TFLOPS, "unit": "TFLOP/s", "frac": op_tf / FP32_FMA_TFLOPS,
                               "peak_source": "H100 SXM data sheet (FP32)"}
        if world == 1 and not a.no_cpu:
            torch.set_num_threads(min(32, os.cpu_count() or 1))
            hs, ws = 270, 480
            small = OF.synthetic_clip(2, hs, ws, seed=7).permute(0, 3, 1, 2).contiguous()
            OS.network_forward(sd, small[0:1], small[1:2])
            t0 = time.perf_counter()
            OS.network_forward(sd, small[0:1], small[1:2])
            sec = time.perf_counter() - t0
            fps = 1.0 / (sec * px / (hs * ws))
            line["cpu_baseline"] = {"value": fps, "unit": "frames/s", "cores": torch.get_num_threads(), "kind": "port",
                                    "sample": f"one {hs}x{ws} pair ({sec:.1f} s) scaled by pixel count to {H}x{W}; oracle/sepconv.py == "
                                              "the reference's PyTorch-CPU path with its op restated on the CPU"}
        print(json.dumps(line))
    eng.close()
    if dist is not None:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
