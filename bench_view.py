"""Measures the sampling network's view (option "sampling_view", the C++ viewer's render-oracle mode) against the full render
on the reference's two shipped trained models (tests/golden/shipped/: Barbershop K = 4, Pavillon K = 16), 800 x 800 frames
through adn_render_camera_rgba8 (the viewer's pixel path).

Per model and mode: frames/s over --steps timed frames (CUDA events around the frames, after --warmup frames), and the
device ms of each stage of one profiled frame (adn_set_option "profile"; slots 0-1 = stage 0 and the sampling MLP,
slot 5 = the view kernel in view mode).  For the view kernel also its achieved bytes/s: it must read raw0 (512 B per ray)
and write one uchar4 (4 B per ray), over its profiled time, against the H100 SXM data sheet's 3.35 TB/s of HBM3.
Prints one JSON line (with the card's name and power limit); writes nothing unless --out is given.

usage: python bench_view.py [--steps K] [--warmup W] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

W = H = 800
HBM_BYTES_PER_S = 3.35e12            # H100 SXM data sheet, HBM3
VIEW_BYTES_PER_RAY = 128 * 4 + 4     # raw0 row in, one uchar4 out
MODELS = {   # shipped export, a pose inside its view cell (offset from the centre, yaw in degrees)
    "barbershop_k4": ([0.3, -0.2, 0.08], 35.0),
    "pavillon_k16": ([0.05, -0.03, 0.02], 0.0),
}
RX = torch.tensor([[1, 0, 0], [0, 0, -1], [0, 1, 0]], dtype=torch.float32)   # camera -z -> world +y


def export_dir(name, dst):
    """Reassembles tests/golden/shipped/<name> (files above 1 MB are split into parts) under dst."""
    src = os.path.join(ROOT, "tests", "golden", "shipped", name)
    with open(os.path.join(src, "manifest.json")) as f:
        man = json.load(f)
    os.makedirs(dst, exist_ok=True)
    for fname, e in man["files"].items():
        with open(os.path.join(dst, fname), "wb") as out:
            for p in e.get("parts", [fname]):
                with open(os.path.join(src, p), "rb") as f:
                    out.write(f.read())
    return dst


def card():
    info = dict(name=torch.cuda.get_device_name(0), power_limit_w=None)
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_w"] = float(r.stdout.strip().splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.TimeoutExpired):
        pass
    return info


def measure(r, pose, rot, thr, K, steps, warmup, view):
    r.set_option("sampling_view", int(view))
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
    # one profiled frame in a run of its own (event records between the stages), as one chunk: a profile times a call's
    # first chunk, and the automatic chunk holds fewer rays than the frame at K = 16
    r.set_option("chunk_rays", W * H)
    r.set_option("profile", 1)
    r.render_camera_rgba8(pose, rot, W, H, thr, K, out=out)
    st = r.stats()
    r.set_option("profile", 0)
    r.set_option("chunk_rays", 0)
    res = dict(ms_per_frame=ms, fps=1000.0 / ms, ms_stage=[round(x, 4) for x in st["ms_stage"]], n_samples=st["n_samples"])
    if view:
        kms = st["ms_stage"][5]
        bps = W * H * VIEW_BYTES_PER_RAY / (kms * 1e-3)
        res.update(view_kernel_ms=kms, view_kernel_bytes_per_s=bps, view_kernel_share_of_hbm=bps / HBM_BYTES_PER_S)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_view.py needs a CUDA device (an H100)")
    from adanerf_b200 import Renderer
    from adanerf_b200.convert import read_dataset_info
    result = dict(bench="sampling_view", frame=f"{W}x{H}", entry="adn_render_camera_rgba8", steps=args.steps, card=card(), models={})
    with tempfile.TemporaryDirectory() as tmp:
        for name, (off, yaw) in MODELS.items():
            d = export_dir(name, os.path.join(tmp, name))
            r, thr, K = Renderer.from_export_dir(d)
            info = read_dataset_info(os.path.join(d, "dataset_info.txt"))
            pose = torch.tensor(info["view_cell_center"], dtype=torch.float32) + torch.tensor(off)
            c, s = torch.cos(torch.deg2rad(torch.tensor(yaw))), torch.sin(torch.deg2rad(torch.tensor(yaw)))
            rot = torch.tensor([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]]) @ RX
            full = measure(r, pose, rot, thr, K, args.steps, args.warmup, view=False)
            view = measure(r, pose, rot, thr, K, args.steps, args.warmup, view=True)
            result["models"][name] = dict(K=K, thr=thr, full=full, view=view)
            r.close()
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
