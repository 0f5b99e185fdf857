"""Measures the fixed-K sampler (option "sampler" = 1, rayMarchSampler FromClassifiedDepth: DONeRF's baseline) next to the
adaptive path on the same networks, at the same K: the reference's shipped Pavillon networks (tests/golden/shipped/
pavillon_k16) used as a DONeRF pair with the sigmoid transform, 800 x 800 frames through adn_render_camera_rgba8 (the
viewer's pixel path), K in {2, 4, 8, 16}.  The adaptive path renders at the export's threshold.

Per K and sampler: frame ms over --steps timed frames (CUDA events, after --warmup frames), samples per frame, and the
device ms of each stage of one profiled frame (slot 2 = the sampler).  For the fixed-K sampler also its achieved bytes/s:
it must read raw0 (512 B per ray) and write z and the ray index (8 B per sample) and count / offset (8 B per ray), over its
profiled time, against the H100 SXM data sheet's 3.35 TB/s of HBM3.  Prints one JSON line per K (with the card's name and
power limit); writes nothing unless --out is given.

usage: python bench_donerf.py [--steps S] [--warmup W] [--out FILE]"""
import argparse
import json
import os
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_view import RX, card, export_dir   # noqa: E402

W = H = 800
KS = (2, 4, 8, 16)
HBM_BYTES_PER_S = 3.35e12            # H100 SXM data sheet, HBM3


def measure(r, pose, rot, thr, K, steps, warmup):
    out = torch.empty((W * H, 4), dtype=torch.uint8, device="cuda")
    for _ in range(warmup):
        r.render_camera_rgba8(pose, rot, W, H, thr, K, out=out)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(steps):
        r.render_camera_rgba8(pose, rot, W, H, thr, K, out=out)
    t1.record()
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / steps
    # one profiled frame in a run of its own, as one chunk (a profile times a call's first chunk), after one unprofiled frame
    # of that chunking, so that growing the scratch buffers to a whole frame is not inside the timed stages
    r.set_option("chunk_rays", W * H)
    r.render_camera_rgba8(pose, rot, W, H, thr, K, out=out)
    r.set_option("profile", 1)
    r.render_camera_rgba8(pose, rot, W, H, thr, K, out=out)
    st = r.stats()
    r.set_option("profile", 0)
    r.set_option("chunk_rays", 0)
    return dict(ms_per_frame=round(ms, 4), fps=round(1000.0 / ms, 2), samples_per_frame=st["n_samples"],
                ms_stage=[round(x, 4) for x in st["ms_stage"]])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_donerf.py needs a CUDA device (an H100)")
    from adanerf_b200 import Renderer
    from adanerf_b200.convert import read_dataset_info
    lines = []
    info_card = card()
    with tempfile.TemporaryDirectory() as tmp:
        d = export_dir("pavillon_k16", os.path.join(tmp, "pavillon_k16"))
        r, thr, _ = Renderer.from_export_dir(d)
        info = read_dataset_info(os.path.join(d, "dataset_info.txt"))
        pose = torch.tensor(info["view_cell_center"], dtype=torch.float32) + torch.tensor([0.05, -0.03, 0.02])
        for K in KS:
            r.set_option("sampler", 1)
            r.set_option("pdf_transform", 1)
            fixed = measure(r, pose, RX, thr, K, args.steps, args.warmup)
            sampler_ms = fixed["ms_stage"][2]
            bps = W * H * (512 + 8 + 8 * K) / (sampler_ms * 1e-3) if sampler_ms > 0 else None
            fixed.update(sampler_bytes_per_s=bps, sampler_share_of_hbm=bps / HBM_BYTES_PER_S if bps else None)
            r.set_option("sampler", 0)
            adaptive = measure(r, pose, RX, thr, K, args.steps, args.warmup)
            lines.append(json.dumps(dict(bench="donerf", frame=f"{W}x{H}", entry="adn_render_camera_rgba8", nets="pavillon_k16",
                                         K=K, thr_adaptive=thr, steps=args.steps, card=info_card, fixed_k=fixed,
                                         adaptive=adaptive)))
            print(lines[-1], flush=True)
        r.close()
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
