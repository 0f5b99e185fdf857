"""Times 800 x 800 frames of sampling nets with D = 32, 64, 128 and 256 depth cells (multiDepthFeatures) at the same K and
threshold: reference-initialised "shaped" nets (oracle/cells_oracle.make_weights, rays ragged at about D / 16 cells over the
threshold).  For each D it reports the median over --reps of
  * stage 2 alone on the frame's raw0 [640000, D] (adn_stage2_sample),
  * the sample-budget select alone (adn_budget_threshold, B = half of the frame's unbudgeted samples),
  * a whole frame (adn_render_camera_rgba8),
each --steps calls between two CUDA events after --warmup calls.  D = 128 runs the existing kernels, so its row is the
baseline the others compare with.  Prints one JSON line per D with the card's name and power limit; writes nothing.

usage: python bench_cells.py [--steps S] [--warmup W] [--reps R] [--K K] [--thr T]"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_view import card   # noqa: E402

W = H = 800


def time_ms(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--K", type=int, default=16)
    ap.add_argument("--thr", type=float, default=0.2)
    a = ap.parse_args(argv)
    import __graft_entry__
    __graft_entry__.build()
    from adanerf_b200 import Renderer
    from oracle import adanerf_oracle as orc
    from oracle import cells_oracle as co
    info = card()
    scene = orc.SCENE_BARBERSHOP
    pose, rot = torch.tensor(scene["view_cell_center"]), orc.rotation_yaw(30.0)
    for D in co.DEPTH_CELLS:
        sd0, sd1 = co.make_weights(D, "shaped", seed=0, thr=a.thr)
        r = Renderer(scene, device=0, sampling_net=sd0, shading_net=sd1)
        x0, _, _ = r.stage0(pose, rot, r.generate_ray_directions(W, H))
        raw0 = r.mlp0(x0)
        del x0
        samples = int(r.stage2(raw0, a.thr, a.K)["total"])
        B = W * H + (samples - W * H) // 2
        thr_out = torch.empty((1,), dtype=torch.float32, device="cuda")
        px = torch.empty((W * H, 4), dtype=torch.uint8, device="cuda")
        rows = {"stage2_ms": [], "budget_ms": [], "frame_ms": []}
        for _ in range(a.reps):
            rows["stage2_ms"].append(time_ms(lambda: r.stage2(raw0, a.thr, a.K), a.steps, a.warmup))
            rows["budget_ms"].append(time_ms(lambda: r.budget_threshold(raw0, a.thr, a.K, B, out=thr_out), a.steps, a.warmup))
            rows["frame_ms"].append(time_ms(lambda: r.render_camera_rgba8(pose, rot, W, H, a.thr, a.K, out=px), a.steps, a.warmup))
        res = dict(bench="cells", D=D, K=a.K, thr=a.thr, W=W, H=H, samples=samples, budget=B, gpu=info["name"],
                   power_limit_w=info["power_limit_w"], **{k: round(statistics.median(v), 4) for k, v in rows.items()},
                   spread={k: [round(min(v), 4), round(max(v), 4)] for k, v in rows.items()})
        print(json.dumps(res), flush=True)
        r.close()


if __name__ == "__main__":
    main()
