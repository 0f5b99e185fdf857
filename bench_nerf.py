"""Measures plain NeRF (option "sampler" = 2, rayMarchSampler LinearlySpacedZNearZFar: K evenly spaced samples on every ray,
no sampling net) next to the adaptive path: the reference's shipped Pavillon networks (tests/golden/shipped/pavillon_k16),
its shading net used as the one NeRF net of a one-network export written beside it (same scene), 800 x 800 frames through adn_render_camera_rgba8 (the viewer's pixel path),
K in {32, 64, 128}.  The adaptive path renders both nets at the export's threshold and K.

Per row: frame ms over --steps timed frames (CUDA events, after --warmup frames), samples per frame, the device ms of each
stage of one profiled frame (slot 0 = rays, 2 = placement, 4 = shading MLP, 5 = composite) and the shading MLP's achieved
TFLOP/s: the dense FLOPs of one NeRF forward (2 x the weights of every layer, from the tensor shapes) times the samples,
over its profiled time.  Prints one JSON line per row (with the card's name and power limit); writes nothing unless --out is
given.

usage: python bench_nerf.py [--steps S] [--warmup W] [--out FILE]"""
import argparse
import json
import os
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_donerf import measure, W, H   # noqa: E402
from bench_view import RX, card, export_dir   # noqa: E402

KS = (32, 64, 128)


def nerf_flops_per_sample(sd):
    """2 x the multiply-adds of one NeRF.forward: every weight matrix once (src/models.py:254-277)."""
    return 2 * sum(int(v.numel()) for k, v in sd.items() if k.endswith(".weight"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_nerf.py needs a CUDA device (an H100)")
    from adanerf_b200 import Renderer
    from adanerf_b200.convert import read_dataset_info
    from adanerf_b200.onnx_weights import write_nerf_export_dir
    from adanerf_b200.synthetic import load_weights_npz
    sd1 = load_weights_npz(os.path.join(ROOT, "tests", "golden", "weights_pavillon"))[1]
    flops = nerf_flops_per_sample({k: torch.as_tensor(v) for k, v in sd1.items()})
    lines = []
    info_card = card()
    with tempfile.TemporaryDirectory() as tmp:
        d = export_dir("pavillon_k16", os.path.join(tmp, "pavillon_k16"))
        adaptive, thr, k_export = Renderer.from_export_dir(d)
        info = read_dataset_info(os.path.join(d, "dataset_info.txt"))
        pose = torch.tensor(info["view_cell_center"], dtype=torch.float32) + torch.tensor([0.05, -0.03, 0.02])
        nd = os.path.join(tmp, "pavillon_nerf")
        write_nerf_export_dir(nd, info, sd1, KS[-1])
        nerf, _, _ = Renderer.from_export_dir(nd)   # one network, option "sampler" = 2
        rows = [("nerf", K) for K in KS] + [("adaptive", k_export)]
        for kind, K in rows:
            r = nerf if kind == "nerf" else adaptive
            m = measure(r, pose, RX, thr, K, args.steps, args.warmup)
            mlp_ms = m["ms_stage"][4]
            m["mlp_tflops"] = round(flops * m["samples_per_frame"] / (mlp_ms * 1e-3) / 1e12, 1) if mlp_ms > 0 else None
            lines.append(json.dumps(dict(bench="nerf", sampler=kind, frame=f"{W}x{H}", entry="adn_render_camera_rgba8",
                                         nets="pavillon_k16 shading net" if kind == "nerf" else "pavillon_k16", K=K,
                                         thr=thr if kind == "adaptive" else None, flops_per_sample=flops, steps=args.steps,
                                         card=info_card, **m)))
            print(lines[-1], flush=True)
        nerf.close()
        adaptive.close()
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
