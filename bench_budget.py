#!/usr/bin/env python
"""bench_budget.py -- frame time under a sample budget (adn_set_option "sample_budget") next to the fixed-threshold frame.

    python bench_budget.py [--workload NAME] [--budget-spr X] [--steps K] [--warmup W] [--gpus N]

One GPU, one 800x800 frame per step through adn_render_camera, the workloads and networks of bench.py.  The workload's
threshold is the floor; the budget is B = round(X * rays per frame).  Prints one JSON line: frames/s and ms per frame of the
fixed-threshold and the budgeted frame (CUDA events around `steps` back-to-back frames each), the chosen threshold, M of both
frames, and the device time of the threshold selection alone (CUDA events over `steps` adn_budget_threshold calls on the
frame's raw0).  Writes nothing into the tree.

--gpus N: the frame in N row bands on devices 0 .. N-1 of one process, through the multi-GPU library (adn_multi_*): the
budget holds for the whole frame and every band renders at the frame's threshold.  Prints the fixed-threshold and the
budgeted frame time (host clock around `steps` frames, each enqueued and waited for), the frame's t* and M, and each band's
M and render time (device events of the last budgeted frame): a shared threshold can load the bands unevenly.
"""
import argparse
import json
import os
import sys

sys.dont_write_bytecode = True   # the tree may be read-only
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def timed(torch, fn, steps, warmup):
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def gpu_and_power_limit(torch):
    import subprocess
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                               text=True, timeout=30).stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return dict(gpu=torch.cuda.get_device_name(0), power_limit=limit)


def run_multi(args, bench, torch):
    import time
    from adanerf_b200 import Renderer, synthetic
    from adanerf_b200.multi import MultiRenderer
    from adanerf_b200.tiling import row_bands
    cfg = bench.WORKLOADS[args.workload]
    W, H, thr, K, G = cfg["W"], cfg["H"], cfg["thr"], cfg["K"], args.gpus
    r, scene, sd0, sd1 = bench.make_renderer_inputs(cfg, torch, Renderer, synthetic, 0, W, H)
    r.close()
    m = MultiRenderer(scene, list(range(G)), sd0, sd1)
    pose, rot = torch.tensor(scene["view_cell_center"], dtype=torch.float32), torch.eye(3)
    budget = int(round(args.budget_spr * W * H))

    def frames(n):
        t0 = time.perf_counter()
        for _ in range(n):
            m.render_camera(pose, rot, W, H, thr, K)
            m.wait_frame()
        return (time.perf_counter() - t0) * 1000.0 / max(n, 1)

    frames(args.warmup)
    fixed_ms = frames(args.steps)
    fixed_m = sum(m.last_samples())
    m.set_option("sample_budget", budget)
    frames(args.warmup)
    budget_ms = frames(args.steps)
    t_star, bands_m = m.last_threshold(), m.last_samples()
    render_ms, gather_ms = m.last_times()
    m.close()
    print(json.dumps(dict(
        workload=args.workload, **gpu_and_power_limit(torch), gpus=G, frame=f"{W}x{H}", K=K, thr_min=thr, steps=args.steps,
        driver="one process, adn_multi_render_camera + adn_multi_wait_frame per frame",
        fixed=dict(threshold=thr, samples=fixed_m, ms_per_frame=fixed_ms, frames_per_s=1000.0 / fixed_ms),
        budget=dict(samples_per_ray=args.budget_spr, max_samples=budget, threshold=t_star, samples=sum(bands_m), ms_per_frame=budget_ms,
                    frames_per_s=1000.0 / budget_ms,
                    bands=[dict(device=i, rows=rows, samples=bm, render_ms=rm, gather_ms=gm)
                           for i, ((_, rows), bm, rm, gm) in enumerate(zip(row_bands(H, G), bands_m, render_ms, gather_ms))]))))


def main():
    import bench
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="800x800_pav_thr0.05_K16", choices=sorted(k for k, c in bench.WORKLOADS.items() if c["thr"] > 0))
    ap.add_argument("--budget-spr", type=float, default=8.0, metavar="X", help="samples per ray of the budget (>= 1)")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--gpus", type=int, default=None, metavar="N", help="the frame in N row bands through the multi-GPU library")
    args = ap.parse_args()
    if args.budget_spr < 1.0:
        raise SystemExit("--budget-spr must be >= 1 (every ray keeps one sample)")
    import torch
    import __graft_entry__ as ge
    ge.build()
    if args.gpus is not None:
        if not 1 <= args.gpus <= torch.cuda.device_count():
            raise SystemExit(f"--gpus {args.gpus}: this machine has {torch.cuda.device_count()} GPUs")
        return run_multi(args, bench, torch)
    from adanerf_b200 import Renderer, synthetic
    cfg = bench.WORKLOADS[args.workload]
    W, H, thr, K = cfg["W"], cfg["H"], cfg["thr"], cfg["K"]
    r, scene, _, _ = bench.make_renderer_inputs(cfg, torch, Renderer, synthetic, 0, W, H)
    pose, rot = torch.tensor(scene["view_cell_center"], dtype=torch.float32), torch.eye(3)
    n = W * H
    budget = int(round(args.budget_spr * n))
    out = torch.empty((n, 3), dtype=torch.float32, device="cuda")

    def frame():
        r.render_camera(pose, rot, W, H, thr, K, out=out)

    fixed_ms = timed(torch, frame, args.steps, args.warmup)
    fixed_m = int(r.render_camera(pose, rot, W, H, thr, K, want_nsamples=True)["n_samples"].long().sum())
    r.set_option("sample_budget", budget)
    budget_ms = timed(torch, frame, args.steps, args.warmup)
    o = r.render_rays(pose, rot, r.generate_ray_directions(W, H), thr, K, want_oracle_weights=True)
    t_star, m = r.last_threshold(), int(o["n_samples"].long().sum())
    t = torch.empty((1,), dtype=torch.float32, device="cuda")
    select_ms = timed(torch, lambda: r.budget_threshold(o["oracle_weights"], thr, K, budget, out=t), args.steps, args.warmup)
    if t.item() != t_star:
        raise SystemExit("the stage-level selection disagrees with the render's")
    r.close()
    print(json.dumps(dict(
        workload=args.workload, gpu=torch.cuda.get_device_name(0), frame=f"{W}x{H}", K=K, thr_min=thr, steps=args.steps,
        fixed=dict(threshold=thr, samples=fixed_m, ms_per_frame=fixed_ms, frames_per_s=1000.0 / fixed_ms),
        budget=dict(samples_per_ray=args.budget_spr, max_samples=budget, threshold=t_star, samples=m, ms_per_frame=budget_ms,
                    frames_per_s=1000.0 / budget_ms, select_ms=select_ms))))


if __name__ == "__main__":
    main()
