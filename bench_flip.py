"""bench_flip.py -- FLIP on the device (adn_image_flip, Renderer.flip): call time, and what the sample budget costs in
image quality.

    python bench_flip.py [--iters N] [--warmup W]

1. Timing.  Pairs of 800 x 800 and 1600 x 1600 Pavillon renders (the two thresholds of one view), per size:
   - call_us:    host wall time per adn_image_flip call, which returns with the mean on the host (N calls after W warm-up);
   - kernel_us:  device time of the three FLIP kernels per call, from torch.profiler in a run of its own;
   - torch_fp32_us: the fp32 torch emulation (oracle/flip_emulation.py, 2-D conv2d filters) on the same GPU, CUDA events;
   - the algorithmic bounds next to them: bytes (two fp32 RGB inputs + the fp32 map) over 3.35 TB/s, and the FP32 FLOP of
     the direct 2-D filters and of the separable ones over 67 TFLOP/s (H100 SXM data sheet, 700 W).
2. Quality.  PSNR and FLIP of Pavillon 800 x 800 renders at thr 0.1 / 0.2 / 0.3 / 0.5 (K = 16) and under sample budgets
   of 4 and 8 samples per ray (floor thr 0.05, K = 16), all against the thr 0.05, K = 16 render: the densest adaptive
   render of the shipped networks, not ground truth.
Prints one JSON line with the card's name and power limit.  Without a GPU it prints that nothing was measured."""
import argparse
import json
import os
import re
import sys
import time

sys.dont_write_bytecode = True   # the tree may be read-only
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

HBM_BYTES_PER_S = 3.35e12
FP32_FLOP_PER_S = 67e12
WORKLOAD = "800x800_pav_thr0.05_K16"


def flop_per_pixel(ppd):
    """FP32 FLOP (2 per MAC) per pixel pair of the filters: 3 CSF channels and 4 feature filters (edge / point in x and y)
    per image, as direct 2-D filters and as the 1-D passes adn_image_flip runs (7 horizontal and 7 vertical per image)."""
    from oracle import flip_emulation as fe
    r, rf = fe.csf_radius(ppd), fe.feature_radius(ppd)
    k, kf = 2 * r + 1, 2 * rf + 1
    direct = 2 * 2 * (3 * k * k + 4 * kf * kf)
    separable = 2 * 2 * (4 * k + 3 * kf + 4 * k + 4 * kf)
    return direct, separable


def bounds(W, H, ppd):
    n = W * H
    direct, separable = flop_per_pixel(ppd)
    t_bytes = n * 28 / HBM_BYTES_PER_S * 1e6
    t_direct = n * direct / FP32_FLOP_PER_S * 1e6
    t_sep = n * separable / FP32_FLOP_PER_S * 1e6
    return dict(bytes=n * 28, flop_direct_2d=n * direct, flop_separable=n * separable, us_bytes_bound=t_bytes,
                us_flop_bound_direct_2d=t_direct, us_flop_bound_separable=t_sep,
                binding_bound_separable="bytes" if t_bytes > t_sep else "FP32 FLOP")


def card(torch):
    import subprocess
    info = dict(name=torch.cuda.get_device_name(0), power_limit_w=None)
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_w"] = float(r.stdout.strip().splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.TimeoutExpired):
        pass
    return info


def time_flip(torch, r, a, b, W, H, iters, warmup):
    import ctypes as C
    from adanerf_b200.renderer import EVALUATE_PPD
    from oracle import flip_emulation as fe
    fmap = torch.empty((H, W), dtype=torch.float32, device="cuda")
    mean = C.c_double()

    def call():
        st = r.lib.adn_image_flip(r.handle, a.data_ptr(), b.data_ptr(), W, H, EVALUATE_PPD, fmap.data_ptr(), C.byref(mean))
        assert st == 0, st
    for _ in range(warmup):
        call()
    t0 = time.perf_counter()
    for _ in range(iters):
        call()
    call_us = (time.perf_counter() - t0) * 1e6 / iters
    # kernel time in a run of its own
    from torch.profiler import ProfilerActivity, profile
    n_prof = min(iters, 20)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n_prof):
            call()
        torch.cuda.synchronize()
    kernels = {}
    for e in prof.key_averages():
        k = re.search(r"flip_\w+_kernel", e.key)
        if k:
            dev = getattr(e, "device_time_total", None)
            if dev is None:
                dev = e.cuda_time_total
            kernels[k.group(0)] = kernels.get(k.group(0), 0.0) + dev / n_prof
    # the fp32 torch emulation, stream ordered on the current stream
    for _ in range(max(1, warmup // 4)):
        fe.flip_map(a, b, W, H, EVALUATE_PPD, torch.float32)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n_torch = max(1, iters // 10)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(n_torch):
        fe.flip_map(a, b, W, H, EVALUATE_PPD, torch.float32)
    e1.record()
    torch.cuda.synchronize()
    torch_us = e0.elapsed_time(e1) * 1e3 / n_torch
    ref32 = fe.flip_map(a, b, W, H, EVALUATE_PPD, torch.float32)
    return dict(call_us=call_us, kernel_us=sum(kernels.values()), kernel_us_each=kernels, torch_fp32_us=torch_us,
                speedup_vs_torch_fp32=torch_us / call_us, mean=mean.value,
                max_abs_diff_vs_torch_fp32=float((fmap - ref32).abs().max()), **bounds(W, H, EVALUATE_PPD))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        print(json.dumps(dict(bench="flip", measured=False, note="not measured: no CUDA device")))
        return
    import __graft_entry__ as ge
    ge.build()
    import bench
    from adanerf_b200 import Renderer, synthetic
    cfg = bench.WORKLOADS[WORKLOAD]
    K, thr_ref = cfg["K"], cfg["thr"]
    r, scene, _, _ = bench.make_renderer_inputs(cfg, torch, Renderer, synthetic, 0, cfg["W"], cfg["H"])
    pose, rot = torch.tensor(scene["view_cell_center"], dtype=torch.float32), torch.eye(3)
    result = dict(bench="flip", measured=True, card=card(torch), workload=WORKLOAD, iters=args.iters, timing={}, quality={})

    for size in (800, 1600):
        a = r.render_camera(pose, rot, size, size, 0.5, K)["rgb"]
        b = r.render_camera(pose, rot, size, size, 0.1, K)["rgb"]
        torch.cuda.synchronize()
        result["timing"][f"{size}x{size}"] = time_flip(torch, r, a, b, size, size, args.iters, args.warmup)

    W = H = 800
    ref = r.render_camera(pose, rot, W, H, thr_ref, K)["rgb"].clone()
    rows = {}
    for thr in (0.1, 0.2, 0.3, 0.5):
        img = r.render_camera(pose, rot, W, H, thr, K, want_nsamples=True)
        rows[f"thr {thr}"] = (img["rgb"], int(img["n_samples"].long().sum()))
    for spr in (4, 8):
        r.set_option("sample_budget", spr * W * H)
        img = r.render_camera(pose, rot, W, H, thr_ref, K, want_nsamples=True)
        rows[f"budget {spr} spr"] = (img["rgb"], int(img["n_samples"].long().sum()))
        r.set_option("sample_budget", 0)
    torch.cuda.synchronize()
    result["quality"]["against"] = f"thr {thr_ref}, K {K} (the densest adaptive render, not ground truth)"
    for name, (img, n_samples) in rows.items():
        m = r.image_metrics(img, ref, clamp01=True)
        f = r.flip(img, ref, W, H, want_map=False)
        result["quality"][name] = dict(samples_per_ray=n_samples / (W * H), psnr_db=m["psnr"], flip=f["mean"])
    r.close()

    print(f"# {result['card']['name']}, power limit {result['card']['power_limit_w']} W")
    for size, t in result["timing"].items():
        print(f"# {size}: adn_image_flip {t['call_us']:.1f} us/call (kernels {t['kernel_us']:.1f} us), torch fp32 "
              f"{t['torch_fp32_us']:.1f} us; bounds: bytes {t['us_bytes_bound']:.1f} us, separable FP32 "
              f"{t['us_flop_bound_separable']:.1f} us, direct 2-D FP32 {t['us_flop_bound_direct_2d']:.1f} us")
    print(f"# quality against {result['quality']['against']}")
    print("# render            spr     PSNR dB   FLIP")
    for name, q in result["quality"].items():
        if name != "against":
            print(f"# {name:16s} {q['samples_per_ray']:6.2f}  {q['psnr_db']:8.3f}  {q['flip']:.5f}")
    print(json.dumps(result))


if __name__ == "__main__":
    main()
