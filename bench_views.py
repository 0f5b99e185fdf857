"""Measures several cameras in one call (adn_render_views_camera_rgba8) against the same views rendered one call each
(adn_render_camera_rgba8), with the reference's shipped Pavillon networks (tests/golden/shipped/pavillon_k16) at the export's
threshold and K:

  (a) a stereo pair of 800 x 800 frames: one views call against two single calls, without and with a sample budget (one B over
      both eyes against B / 2 per eye);
  (b) 64 views of 100 x 100: one views call against 64 calls;
  (c) V = 1: the views entry against the existing single-view entry.

The two sides of each row run alternately in one process, --reps times each, every time --steps groups of calls between
two CUDA events after --warmup groups; a row reports the median ms per group (one frame of V views) of each side and their
ratio.  Prints one JSON line per row with the card's name and power limit; writes nothing unless --out is given.

usage: python bench_views.py [--steps S] [--warmup W] [--reps R] [--out FILE]"""
import argparse
import json
import os
import statistics
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_view import RX, card, export_dir   # noqa: E402


def cameras(center, V):
    """V cameras around the view-cell centre, each a 1 / V turn further (positions and rotations differ)."""
    import math
    poses, rots = [], []
    for v in range(V):
        t = 2 * math.pi * v / V
        poses.append(torch.tensor(center, dtype=torch.float32) + torch.tensor([0.05 * math.cos(t), 0.05 * math.sin(t), 0.0]))
        c, s = math.cos(t), math.sin(t)
        yaw = torch.tensor([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]], dtype=torch.float32)
        rots.append(yaw @ RX)
    return torch.stack(poses), torch.stack(rots)


def time_group(fn, steps, warmup):
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


def compare(one, many, steps, warmup, reps):
    """Median ms per group of the views call (one) and the single calls (many), alternated."""
    t1, tn = [], []
    for _ in range(reps):
        t1.append(time_group(one, steps, warmup))
        tn.append(time_group(many, steps, warmup))
    m1, mn = statistics.median(t1), statistics.median(tn)
    return dict(views_call_ms=round(m1, 4), single_calls_ms=round(mn, 4), speedup=round(mn / m1, 3),
                views_call_ms_all=[round(x, 4) for x in t1], single_calls_ms_all=[round(x, 4) for x in tn])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_views.py needs a CUDA device (an H100)")
    from adanerf_b200 import Renderer
    from adanerf_b200.convert import read_dataset_info
    info_card = card()
    lines = []
    with tempfile.TemporaryDirectory() as tmp:
        d = export_dir("pavillon_k16", os.path.join(tmp, "pavillon_k16"))
        r, thr, K = Renderer.from_export_dir(d)
        center = read_dataset_info(os.path.join(d, "dataset_info.txt"))["view_cell_center"]

        def row(name, V, W, H, budget=0):
            poses, rots = cameras(center, V)
            outs = [torch.empty((W * H, 4), dtype=torch.uint8, device="cuda") for _ in range(V)]

            def one():   # V = 1 too goes through adn_render_views_camera_rgba8
                r.set_option("sample_budget", budget)
                r.render_views_camera(poses, rots, W, H, thr, K, rgba8=True)

            def many():
                r.set_option("sample_budget", budget // V)
                for v in range(V):
                    r.render_camera_rgba8(poses[v], rots[v], W, H, thr, K, out=outs[v])

            res = compare(one, many, args.steps, args.warmup, args.reps)
            r.set_option("sample_budget", 0)
            lines.append(json.dumps(dict(bench="views", row=name, views=V, frame=f"{W}x{H}", K=K, thr=thr,
                                         sample_budget=budget or None, nets="pavillon_k16", steps=args.steps, reps=args.reps,
                                         card=info_card, **res)))
            print(lines[-1], flush=True)

        row("a_stereo", 2, 800, 800)
        row("a_stereo_budget", 2, 800, 800, budget=2 * 800 * 800 * 4)
        row("b_64_small_views", 64, 100, 100)
        row("c_one_view", 1, 800, 800)
        r.close()
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
