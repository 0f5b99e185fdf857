"""TEST INFRASTRUCTURE -- generates tests/golden/flip_*.npz by running the UNMODIFIED reference src/util/flip_loss.py on
CPU in the build container (next to oracle/ref_harness.py, which locates the reference checkout).

    python oracle/gen_flip_golden.py        # rewrites tests/golden/flip_*

The reference module hard-codes the GPU (`.cuda()` on tensors and `torch.zeros(..., device='cuda')`); the run replaces
Tensor.cuda with the identity and gives the module a `torch` whose `zeros` drops the device, and changes nothing else.
Each case is computed twice: with fp32 tensors, as evaluate.py runs it (the fixture's map and mean), and with the default
dtype set to fp64, whose per-pixel distance to the fp32 map is recorded as the reference's own rounding spread.
Every fixture holds the inputs ([H*W, 3] fp32 as evaluate.py holds them), the fp32 map [H, W] and mean, the fp32-vs-fp64
spread, and in its meta the ppd, both radii and cmax.
"""
import json
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import ref_harness as rh          # noqa: E402
from oracle import flip_emulation as fe       # noqa: E402
from oracle.gen_golden import save            # noqa: E402

PPD_CAP = 200.0   # the largest pixels_per_degree adn_image_flip accepts


def _reference_module():
    rh._install_stubs()
    from util import flip_loss
    shim = types.ModuleType("torch_without_cuda")
    shim.__dict__.update(torch.__dict__)
    shim.zeros = lambda *a, device=None, **k: torch.zeros(*a, **k)
    flip_loss.torch = shim
    return flip_loss


def reference_flip(image, reference, W, H, ppd, dtype):
    """The reference's map [H, W] (numpy) and mean, evaluate.py's call: compute_flip(test, reference, ppd) on NCHW views."""
    fl = _reference_module()
    old_cuda, old_dtype = torch.Tensor.cuda, torch.get_default_dtype()
    torch.Tensor.cuda = lambda self, *a, **k: self
    torch.set_default_dtype(dtype)
    try:
        t = torch.from_numpy(image).to(dtype).view(1, H, W, -1).permute(0, 3, 1, 2)
        r = torch.from_numpy(reference).to(dtype).view(1, H, W, -1).permute(0, 3, 1, 2)
        m = fl.FLIP().compute_flip(t, r, ppd)
        assert m.dtype == dtype, m.dtype
        return m[0, 0].numpy(), torch.mean(m).item()
    finally:
        torch.Tensor.cuda = old_cuda
        torch.set_default_dtype(old_dtype)


def write_case(name, image, reference, W, H, ppd=fe.EVALUATE_PPD, **extra):
    image = np.ascontiguousarray(image, np.float32).reshape(H * W, 3)
    reference = np.ascontiguousarray(reference, np.float32).reshape(H * W, 3)
    m32, mean32 = reference_flip(image, reference, W, H, ppd, torch.float32)
    m64, mean64 = reference_flip(image, reference, W, H, ppd, torch.float64)
    assert np.array_equal(np.isnan(m32), np.isnan(m64))
    ok = ~np.isnan(m32)
    spread = float(np.abs(m32[ok].astype(np.float64) - m64[ok]).max()) if ok.any() else 0.0
    meta = dict(W=W, H=H, ppd=ppd, radius_csf=fe.csf_radius(ppd), radius_feature=fe.feature_radius(ppd), cmax=fe.cmax(),
                mean_fp64=mean64, torch_version=torch.__version__,
                generator="oracle/gen_flip_golden.py (unmodified reference util/flip_loss.py, CPU)", **extra)
    save(f"flip_{name}.npz", meta=np.array(json.dumps(meta)), image=image, reference=reference, map=m32.astype(np.float32),
         mean=np.float64(mean32), spread=np.float64(spread))
    print(f"  {name}: {W}x{H} ppd {ppd:.4f} mean {mean32:.8g} spread {spread:.3g}")


def pavillon_renders(W, H, thrs, K=16):
    """Renders of the shipped Pavillon networks by the CPU oracle (oracle/adanerf_oracle.py), one per threshold."""
    from adanerf_b200.synthetic import load_weights_npz
    from oracle import adanerf_oracle as orc
    sd0, sd1 = load_weights_npz(os.path.join(ROOT, "tests", "golden", "weights_pavillon"))
    scene = orc.SCENE_PAVILLON
    rx = torch.tensor([[1, 0, 0], [0, 0, -1], [0, 1, 0]], dtype=torch.float32)
    dirs = torch.from_numpy(orc.generate_ray_directions(W, H, scene["fov"]).reshape(-1, 3)).float()
    pose = torch.tensor(scene["view_cell_center"], dtype=torch.float32) + torch.tensor([0.05, -0.03, 0.02])
    return [orc.render_frame(pose, rx, dirs, sd0, sd1, scene, thr, K)[0].numpy() for thr in thrs]


def main():
    if not rh.available():
        sys.exit("needs the reference checkout (oracle/ref_harness.py)")
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    rng = np.random.default_rng(2020)
    # non-square noise: a W / H transposition cannot pass
    write_case("noise_256x192", rng.random((192, 256, 3)), rng.random((192, 256, 3)), 256, 192)
    # smooth: low-frequency colour fields, the second slightly shifted and tinted
    yy, xx = np.mgrid[0:120, 0:160] / 40.0
    a = np.stack([0.5 + 0.4 * np.sin(xx + 0.3 * yy), 0.5 + 0.4 * np.cos(0.7 * yy), 0.5 + 0.3 * np.sin(xx * yy / 3)], -1)
    b = np.stack([0.5 + 0.4 * np.sin(xx + 0.05 + 0.3 * yy), 0.52 + 0.4 * np.cos(0.7 * yy), 0.47 + 0.3 * np.sin(xx * yy / 3)], -1)
    write_case("smooth_160x120", a, b, 160, 120)
    # edges and points: bars, a checkerboard and isolated dots against the same pattern moved by one pixel
    p = np.zeros((64, 64, 3))
    p[:, 10:12] = 1.0
    p[20:22, :, 1] = 1.0
    p[40:, 40:] = ((np.add.outer(np.arange(24), np.arange(24)) // 3) % 2)[..., None]
    p[5:60:9, 5:60:9] = [1.0, 0.2, 0.7]
    write_case("pattern_64x64", p, np.roll(p, (1, 1), (0, 1)), 64, 64)
    # inputs outside [0, 1], with +-inf
    o1 = rng.uniform(-0.5, 1.5, (40, 48, 3))
    o2 = rng.uniform(-0.5, 1.5, (40, 48, 3))
    o1[3, 4, 0], o1[10, 30, 2], o2[25, 7, 1], o2[39, 47, 0] = np.inf, -np.inf, np.inf, -np.inf
    write_case("outside_48x40", o1, o2, 48, 40)
    # one NaN pixel at (x, y) = (5, 5): NaN over the 16 x 16 block within the CSF radius
    n1, n2 = rng.random((32, 32, 3)), rng.random((32, 32, 3))
    n1[5, 5, 1] = np.nan
    write_case("nan_32x32", n1, n2, 32, 32)
    same = rng.random((24, 40, 3))
    write_case("identical_40x24", same, same, 40, 24)
    write_case("tiny_7x5", rng.random((5, 7, 3)), rng.random((5, 7, 3)), 7, 5)
    write_case("tiny_1x1", rng.random((1, 1, 3)), rng.random((1, 1, 3)), 1, 1)
    # other observers: ppd 30 and the cap
    s1, s2 = 0.7 * a[:48, :64] + 0.3 * rng.random((48, 64, 3)), 0.7 * b[:48, :64] + 0.3 * rng.random((48, 64, 3))
    write_case("ppd30_64x48", s1, s2, 64, 48, ppd=30.0)
    write_case("ppdcap_64x48", s1, s2, 64, 48, ppd=PPD_CAP)
    # real renders: the shipped Pavillon networks at two thresholds
    lo, hi = pavillon_renders(48, 40, (0.1, 0.5))
    write_case("pavillon_48x40", hi, lo, 48, 40, render="oracle, Pavillon K=16, image thr 0.5, reference thr 0.1")


if __name__ == "__main__":
    main()
