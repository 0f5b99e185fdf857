"""bench_iwssim.py -- IW-SSIM on the device (adn_image_iwssim, Renderer.iw_ssim): call time, and what the sample budget
costs in all three of evaluate.py's metrics.

    python bench_iwssim.py [--iters N] [--warmup W]

1. Timing.  Pairs of 800 x 800 and 1600 x 1600 Pavillon renders (two thresholds of one view) in the evaluate layout, per size:
   - call_us:    host wall time per adn_image_iwssim call, which returns with the score on the host (N calls after W warm-up);
   - kernel_us:  device time of the ten IW-SSIM launches per call, from torch.profiler in a run of its own;
   - torch_fp32_us: the fp32 torch emulation (oracle/iwssim_emulation.py: numpy fp64 pyramid on the host, the rest on the
     same GPU), host wall time to its score;
   - bounds from shapes: the bytes the ten kernels move over 3.35 TB/s, and their FP64 work over 34 TFLOP/s (H100 SXM data
     sheet, non-tensor FP64, 700 W).
2. Quality.  PSNR, FLIP and IW-SSIM (evaluate layout, as evaluate.py computes it) of Pavillon 800 x 800 renders at thr
   0.1 / 0.2 / 0.3 / 0.5 (K = 16) and under sample budgets of 4 and 8 samples per ray (floor thr 0.05, K = 16), all against
   the thr 0.05, K = 16 render: the densest adaptive render of the shipped networks, not ground truth.  IW-SSIM on the
   0-255 gray scale of the same renders is printed next to it.
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
FP64_FLOP_PER_S = 34e12
WORKLOAD = "800x800_pav_thr0.05_K16"


def level_sizes(rows, cols, nsc=5):
    out = []
    for _ in range(nsc):
        out.append((rows, cols))
        rows, cols = (rows + 1) // 2, (cols + 1) // 2
    return out


def bounds(W, H):
    """Global bytes and FP64 FLOP (2 per FMA) of the ten launches for a W x H evaluate-layout pair, counted from shapes."""
    lv = level_sizes(W, H)
    n = [r * c for r, c in lv]
    cs = [(r - 10) * (c - 10) for r, c in lv]
    interior = [(r - 2) * (c - 2) for r, c in lv]
    b = 2 * n[0] * 12 + 2 * n[0] * 8                                   # gray: RGB in, fp64 level 0 out
    b += sum(2 * (n[l] + n[l + 1]) * 8 for l in range(4))              # reductions
    b += sum(2 * (n[l] + (n[l + 1] if l < 4 else 0)) * 8 + 2 * n[l] * 4 for l in range(5))   # bands
    b += sum(n[s] * 4 + n[s + 1] * 4 for s in range(4))                # covariance: original band and parent
    b += sum(2 * n[s] * 4 for s in range(5))                           # quality and weights: both bands
    f = sum(2 * n[l + 1] * 2 * 30 for l in range(4))                   # 5 x 5 + 5 taps per reduced sample
    f += sum(2 * n[l] * 2 * 12 for l in range(4))                      # <= 9 nonzero upConv taps + 3
    f += sum(interior[s] * 2 * (55 + 24) for s in range(4))            # Y^T Y entries, parent interpolation
    h = 2 * 5 * 11 + 5                                                 # one 1-D pass of five moment planes
    f += sum(cs[s] * (18 / 8 * h + h + 10) for s in range(5))          # separable statistics, cs / l
    f += sum(cs[s] * (2 * 45 + 2 * 110 + 10 * 25 + 40) for s in range(4))   # 3 x 3 stats, y^T C^-1 y, 10 log2, infow
    t_bytes, t_flop = b / HBM_BYTES_PER_S * 1e6, f / FP64_FLOP_PER_S * 1e6
    return dict(bytes=b, fp64_flop=f, us_bytes_bound=t_bytes, us_fp64_bound=t_flop,
                binding_bound="bytes" if t_bytes > t_flop else "FP64 FLOP")


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


def time_iwssim(torch, r, a, b, W, H, iters, warmup):
    import ctypes as C
    from oracle import iwssim_emulation as ie
    score, scales = C.c_double(), (C.c_double * 5)()

    def call():
        st = r.lib.adn_image_iwssim(r.handle, a.data_ptr(), b.data_ptr(), W, H, 1, C.byref(score), scales)
        assert st == 0, st
    for _ in range(warmup):
        call()
    t0 = time.perf_counter()
    for _ in range(iters):
        call()
    call_us = (time.perf_counter() - t0) * 1e6 / iters
    from torch.profiler import ProfilerActivity, profile
    n_prof = min(iters, 20)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n_prof):
            call()
        torch.cuda.synchronize()
    kernels = {}
    for e in prof.key_averages():
        k = re.search(r"iwssim_\w+_kernel", e.key)
        if k:
            dev = getattr(e, "device_time_total", None)
            if dev is None:
                dev = e.cuda_time_total
            kernels[k.group(0)] = kernels.get(k.group(0), 0.0) + dev / n_prof
    o, d = ie.metric_images(a, b, W, H, "evaluate")
    ie.iwssim(o, d, torch.float32, device="cuda")
    n_torch = 3
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n_torch):
        e32 = ie.iwssim(o, d, torch.float32, device="cuda")
    torch.cuda.synchronize()
    torch_us = (time.perf_counter() - t0) * 1e6 / n_torch
    return dict(call_us=call_us, kernel_us=sum(kernels.values()), kernel_us_each=kernels, torch_fp32_us=torch_us,
                speedup_vs_torch_fp32=torch_us / call_us, score=score.value, scales=list(scales),
                score_torch_fp32=e32["score"], **bounds(W, H))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        print(json.dumps(dict(bench="iwssim", measured=False, note="not measured: no CUDA device")))
        return
    import __graft_entry__ as ge
    ge.build()
    import bench
    from adanerf_b200 import Renderer, synthetic
    cfg = bench.WORKLOADS[WORKLOAD]
    K, thr_ref = cfg["K"], cfg["thr"]
    r, scene, _, _ = bench.make_renderer_inputs(cfg, torch, Renderer, synthetic, 0, cfg["W"], cfg["H"])
    pose, rot = torch.tensor(scene["view_cell_center"], dtype=torch.float32), torch.eye(3)
    result = dict(bench="iwssim", measured=True, card=card(torch), workload=WORKLOAD, iters=args.iters, timing={}, quality={})

    for size in (800, 1600):
        a = r.render_camera(pose, rot, size, size, 0.5, K)["rgb"]
        b = r.render_camera(pose, rot, size, size, 0.1, K)["rgb"]
        torch.cuda.synchronize()
        result["timing"][f"{size}x{size}"] = time_iwssim(torch, r, a, b, size, size, args.iters, args.warmup)

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

    def gray255(x):
        return (255 * (0.2989 * x[:, 0] + 0.5870 * x[:, 1] + 0.1140 * x[:, 2])).contiguous()
    result["quality"]["against"] = f"thr {thr_ref}, K {K} (the densest adaptive render, not ground truth)"
    for name, (img, n_samples) in rows.items():
        m = r.image_metrics(img, ref, clamp01=True)
        f = r.flip(img, ref, W, H, want_map=False)
        s = r.iw_ssim(img, ref, W, H)
        g = r.iw_ssim(gray255(img), gray255(ref), W, H, layout="gray")
        result["quality"][name] = dict(samples_per_ray=n_samples / (W * H), psnr_db=m["psnr"], flip=f["mean"],
                                       iw_ssim=s["score"], iw_ssim_gray255=g["score"])
    r.close()

    print(f"# {result['card']['name']}, power limit {result['card']['power_limit_w']} W")
    for size, t in result["timing"].items():
        print(f"# {size}: adn_image_iwssim {t['call_us']:.1f} us/call (kernels {t['kernel_us']:.1f} us), torch fp32 "
              f"{t['torch_fp32_us']:.1f} us; bounds: bytes {t['us_bytes_bound']:.1f} us, FP64 {t['us_fp64_bound']:.1f} us")
        for k, v in sorted(t["kernel_us_each"].items(), key=lambda kv: -kv[1]):
            print(f"#     {k:22s} {v:8.1f} us")
    print(f"# quality against {result['quality']['against']}")
    print("# render            spr     PSNR dB   FLIP     IW-SSIM   IW-SSIM (gray 0-255)")
    for name, q in result["quality"].items():
        if name != "against":
            print(f"# {name:16s} {q['samples_per_ray']:6.2f}  {q['psnr_db']:8.3f}  {q['flip']:.5f}  {q['iw_ssim']:.6f}  "
                  f"{q['iw_ssim_gray255']:.6f}")
    print(json.dumps(result))


if __name__ == "__main__":
    main()
