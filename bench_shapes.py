#!/usr/bin/env python
"""bench_shapes.py -- frame time of networks of other shapes than 8 x 256 / skip 4, next to the default networks.

    python bench_shapes.py [--steps K] [--warmup W] [--repeats R] [--encodings]

One GPU, one 800x800 frame per step through adn_render_camera (Barbershop geometry, camera at the view-cell centre), for
every (sampling net, shading net) pair of the grid below and two workloads: thr 0.2 / K = 8, and a ragged thr 0.05 /
K = 16 case like the Pavillon workload of bench.py (1..16 samples per ray).  The networks are
oracle/shape_oracle.make_shape_weights of the shape.  Every shape is warmed up first; then, `repeats` times, the control
(8 x 256 / 8 x 256 skip 4) and each other shape are timed back to back, alternating.  Prints one JSON line per shape and
workload: frames/s (min / median / max over the repeats) and the control's next to it, per-stage device ms of one profiled
frame, the MLPs' achieved TFLOP/s from the algorithmic FLOPs of the unpadded networks, and the card and its power limit
read in the same run.  Writes nothing into the tree.

--encodings: the positional-encoding grid ENC_GRID instead (8 x 256 nets, posEncArgs as listed, timed next to the 10-4
control the same way); the weights are oracle/gen_encoding_golden.encoding_weights of the encoding.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.dont_write_bytecode = True   # the tree may be read-only
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

W = H = 800
# (sampling layers, width), (shading layers, width, skips entry) -- the control first
GRID = [((8, 256), (8, 256, "auto")), ((8, 256), (8, 128, "auto")), ((8, 256), (6, 128, "3")), ((8, 256), (4, 256, "auto")),
        ((8, 256), (10, 256, "auto")), ((6, 128), (8, 256, "auto")), ((6, 128), (6, 128, "3"))]
# (sampling bands (P0, D0), shading bands (P, D), label) -- the control first; posEnc none = (-1, -1)
ENC_GRID = [((10, 4), (10, 4), "10-4 / 10-4"), ((10, 4), (15, 4), "10-4 / 15-4"), ((10, 4), (20, 10), "10-4 / 20-10"),
            ((10, 4), (-1, -1), "10-4 / none"), ((16, 4), (10, 4), "16-4 / 10-4")]
WORKLOADS = {"thr0.2_K8": dict(thr=0.2, K=8, target_spr=8.0), "ragged_thr0.05_K16": dict(thr=0.05, K=16, target_spr=10.0)}


def sampling_macs(D, Wd, n_in=90, n_out=128):
    """Multiply-adds per ray of BaseNet(D, W): n_in -> W, D - 2 times W -> W, W -> n_out."""
    return n_in * Wd + (D - 2) * Wd * Wd + Wd * n_out if D > 1 else n_in * Wd


def shading_macs(D, Wd, skip, n_p=63, n_v=27):
    """Multiply-adds per sample of NeRF(D, W, skip, use_viewdirs) reading n_p position and n_v view columns (63 and 27 for
    posEnc 10-4): the pts layers (the skip consumer reads W + n_p), feature, alpha, the view layer (W + n_v -> W/2) and rgb."""
    pts = n_p * Wd + sum((Wd + n_p if i == skip + 1 and skip >= 0 else Wd) * Wd for i in range(1, D))
    return pts + Wd * Wd + Wd + (Wd + n_v) * (Wd // 2) + 3 * (Wd // 2)


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--encodings", action="store_true", help="time the positional-encoding grid ENC_GRID")
    args = ap.parse_args()
    import torch
    import __graft_entry__ as ge
    ge.build()
    from adanerf_b200 import Renderer
    from oracle import adanerf_oracle as orc
    from oracle import shape_oracle as so
    gpu, limit = torch.cuda.get_device_name(0), power_limit_w()
    scene = orc.SCENE_BARBERSHOP
    pose, rot = torch.tensor(scene["view_cell_center"], dtype=torch.float32), torch.eye(3)
    out = torch.empty((W * H, 3), dtype=torch.float32, device="cuda")

    def timed(r, thr, K):
        for _ in range(args.warmup):
            r.render_camera(pose, rot, W, H, thr, K, out=out)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(args.steps):
            r.render_camera(pose, rot, W, H, thr, K, out=out)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.steps

    if args.encodings:
        return encodings(args, timed, scene, pose, rot, out, gpu, limit)
    for wname, wl in WORKLOADS.items():
        thr, K = wl["thr"], wl["K"]
        renderers = []
        for (d0, w0), (d1, w1, skip) in GRID:
            sd0, sd1 = so.make_shape_weights((d0, d1), (w0, w1), skip, thr=thr, target_spr=wl["target_spr"])
            r = Renderer(scene, device=0, sampling_net=sd0, shading_net=sd1)
            r.set_option("chunk_rays", W * H)   # one chunk: the profiled stage times cover the whole frame
            timed(r, thr, K)                    # warm-up of every shape
            renderers.append(r)
        ms = [[] for _ in GRID]
        ctrl_ms = [[] for _ in GRID]
        for _ in range(args.repeats):
            for i, r in enumerate(renderers):
                ctrl_ms[i].append(timed(renderers[0], thr, K))
                ms[i].append(timed(r, thr, K))
        for i, ((d0, w0), (d1, w1, skip)) in enumerate(GRID):
            r = renderers[i]
            r.set_option("profile", 1)
            r.render_camera(pose, rot, W, H, thr, K, out=out)
            st = r.stats()
            r.set_option("profile", 0)
            s1 = r.net_shape(1)
            m = st["n_samples"]
            f0, f1 = 2.0 * sampling_macs(d0, w0) * W * H, 2.0 * shading_macs(*s1) * m
            ms0, ms1 = st["ms_stage"][1], st["ms_stage"][4]
            fps = sorted(1000.0 / t for t in ms[i])
            cfps = sorted(1000.0 / t for t in ctrl_ms[i])
            print(json.dumps(dict(
                workload=f"{W}x{H}_{wname}", gpu=gpu, power_limit_w=limit, steps=args.steps, repeats=args.repeats,
                sampling=dict(layers=d0, width=w0, shape=list(r.net_shape(0)), mac_per_ray=sampling_macs(d0, w0)),
                shading=dict(layers=d1, width=w1, skips=skip, shape=list(s1), mac_per_sample=shading_macs(*s1)),
                samples=m, samples_per_ray=m / (W * H),
                frames_per_s=dict(min=fps[0], median=statistics.median(fps), max=fps[-1]),
                control_frames_per_s=dict(min=cfps[0], median=statistics.median(cfps), max=cfps[-1]),
                ms_stage=[round(x, 4) for x in st["ms_stage"]],
                tflops=dict(sampling_mlp=f0 / (ms0 * 1e9) if ms0 > 0 else None, shading_mlp=f1 / (ms1 * 1e9) if ms1 > 0 else None))))
            sys.stdout.flush()
        for r in renderers:
            r.close()


def encodings(args, timed, scene, pose, rot, out, gpu, limit):
    from adanerf_b200 import Renderer
    from oracle import gen_encoding_golden as geg
    for wname, wl in WORKLOADS.items():
        thr, K = wl["thr"], wl["K"]
        renderers = []
        for b0, b1, _ in ENC_GRID:
            sc = dict(scene, n_freq_pos=b1[0], n_freq_dir=b1[1], n_freq_pos0=b0[0] or -1, n_freq_dir0=b0[1] or -1)
            sd0, sd1 = geg.encoding_weights(b0, tuple(max(x, 0) for x in b1), (8, 256, "auto"), thr, wl["target_spr"], sc)
            r = Renderer(sc, device=0, sampling_net=sd0, shading_net=sd1)
            r.set_option("chunk_rays", W * H)
            timed(r, thr, K)
            renderers.append(r)
        ms, ctrl_ms = [[] for _ in ENC_GRID], [[] for _ in ENC_GRID]
        for _ in range(args.repeats):
            for i, r in enumerate(renderers):
                ctrl_ms[i].append(timed(renderers[0], thr, K))
                ms[i].append(timed(r, thr, K))
        for i, (b0, b1, label) in enumerate(ENC_GRID):
            r = renderers[i]
            r.set_option("profile", 1)
            r.render_camera(pose, rot, W, H, thr, K, out=out)
            st = r.stats()
            r.set_option("profile", 0)
            m = st["n_samples"]
            n0, n_p, n_v = 6 + 6 * (b0[0] + b0[1]), 3 + 6 * max(b1[0], 0), 3 + 6 * max(b1[1], 0)
            f0, f1 = 2.0 * sampling_macs(8, 256, n_in=n0) * W * H, 2.0 * shading_macs(8, 256, 4, n_p, n_v) * m
            ms0, ms1 = st["ms_stage"][1], st["ms_stage"][4]
            fps, cfps = sorted(1000.0 / t for t in ms[i]), sorted(1000.0 / t for t in ctrl_ms[i])
            print(json.dumps(dict(
                workload=f"{W}x{H}_{wname}", gpu=gpu, power_limit_w=limit, steps=args.steps, repeats=args.repeats,
                encoding=label, columns=dict(sampling=n0, position=n_p, view=n_v), samples=m, samples_per_ray=m / (W * H),
                frames_per_s=dict(min=fps[0], median=statistics.median(fps), max=fps[-1]),
                control_frames_per_s=dict(min=cfps[0], median=statistics.median(cfps), max=cfps[-1]),
                ms_stage=[round(x, 4) for x in st["ms_stage"]],
                tflops=dict(sampling_mlp=f0 / (ms0 * 1e9) if ms0 > 0 else None, shading_mlp=f1 / (ms1 * 1e9) if ms1 > 0 else None))))
            sys.stdout.flush()
        for r in renderers:
            r.close()


if __name__ == "__main__":
    main()
