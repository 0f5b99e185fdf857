"""TEST INFRASTRUCTURE -- generates tests/golden/iwssim_* by running the UNMODIFIED reference src/util/IW_SSIM_PyTorch.py on
CPU in the build container (next to oracle/ref_harness.py, which locates the reference checkout).

    python oracle/gen_iwssim_golden.py        # rewrites tests/golden/iwssim_*

The reference module cannot run as shipped on current torch: it imports pyrtools, and it calls torch.eig, which torch 2
removed.  The run changes exactly three things:
  * sys.modules["pyrtools"] is a module whose pyramids.LaplacianPyramid is oracle/laplacian_pyramid.py's restatement;
  * torch.eig is an adapter over torch.linalg.eig returning the old [n, 2] (real, imaginary) eigenvalues and the real
    eigenvectors;
  * the class is constructed with use_cuda=False.
Each case runs the class twice, with use_double=False (evaluate.py's fp32 path: the fixture's score) and use_double=True;
their difference is the reference's own rounding spread.  Every fixture holds the inputs as the caller passes them to
adn_image_iwssim (layout "gray": [H*W] planes on the 0-255 scale; "evaluate": [H*W, 3] as evaluate.py holds them), the
metric's 2-D images (the evaluate-layout conversion, bit for bit), both reference scores and wmcs, and the fp64 emulation's five
wmcs and score (oracle/iwssim_emulation.py).
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

from oracle import ref_harness as rh             # noqa: E402
from oracle import iwssim_emulation as ie        # noqa: E402
from oracle import laplacian_pyramid as lp       # noqa: E402
from oracle.gen_golden import save               # noqa: E402


class _Pyramid:
    def __init__(self, image, height):
        self.pyr_coeffs = {(i, 0): b for i, b in enumerate(lp.laplacian_pyramid(image, height))}


def _eig(a, eigenvectors=False):
    w, v = torch.linalg.eig(a)
    vals = torch.stack([w.real, w.imag], 1)
    return vals, (v.real if eigenvectors else torch.empty(0, dtype=a.dtype))


def _reference_class():
    rh._install_stubs()
    pyr = types.ModuleType("pyrtools")
    pyr.pyramids = types.SimpleNamespace(LaplacianPyramid=lambda image, height=5: _Pyramid(image, height))
    sys.modules["pyrtools"] = pyr
    torch.eig = _eig
    from util.IW_SSIM_PyTorch import IW_SSIM
    return IW_SSIM


def reference_score(original, distorted, use_double):
    """The reference's score of two 2-D numpy images (original, distorted) from its test(), and its five wmcs from its
    own stages (test() keeps them local), or NaNs where its torch.inverse raises."""
    ref = _reference_class()(use_cuda=False, use_double=use_double)
    try:
        score = float(ref.test(original.copy(), distorted.copy()))
        dt = np.float64 if use_double else np.float32
        po, pd = ref.get_pyrd(original.astype(dt), distorted.astype(dt))
        lmap, cs = ref.scale_qualty_maps(po, pd)
        iw = ref.info_content_weight_map(po, pd)
    except RuntimeError:
        return float("nan"), [float("nan")] * ie.NSC
    b = ie.BOUND1
    wmcs = [float(torch.sum(cs[s] * iw[s][:, :, b:-b, b:-b]) / torch.sum(iw[s][:, :, b:-b, b:-b])) for s in range(1, ie.NSC)]
    return score, wmcs + [float(torch.mean(cs[ie.NSC] * lmap))]


def write_case(name, image, reference, W, H, layout, **extra):
    if layout == "evaluate":
        image = np.ascontiguousarray(image, np.float32).reshape(H * W, 3)
        reference = np.ascontiguousarray(reference, np.float32).reshape(H * W, 3)
    else:
        image = np.ascontiguousarray(image, np.float32).reshape(H * W)
        reference = np.ascontiguousarray(reference, np.float32).reshape(H * W)
    orig, dist = ie.metric_images(torch.from_numpy(image), torch.from_numpy(reference), W, H, layout)
    orig, dist = orig.numpy(), dist.numpy()
    ref32, wmcs32 = reference_score(orig, dist, False)
    ref64, wmcs64 = reference_score(orig, dist, True)
    emu = ie.iwssim(orig, dist, torch.float64)
    meta = dict(W=W, H=H, layout=layout, score_fp32=ref32, score_fp64=ref64, wmcs_fp32=wmcs32, wmcs_fp64=wmcs64,
                torch_version=torch.__version__,
                generator="oracle/gen_iwssim_golden.py (unmodified reference util/IW_SSIM_PyTorch.py, CPU)", **extra)
    save(f"iwssim_{name}.npz", meta=np.array(json.dumps(meta)), image=image, reference=reference, original=orig,
         distorted=dist, wmcs_emulation=np.array(emu["wmcs"], np.float64), score_emulation=np.float64(emu["score"]))
    print(f"  {name}: {W}x{H} {layout} ref32 {ref32:.10g} ref64 {ref64:.10g} emulation {emu['score']:.10g}")


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
    rng = np.random.default_rng(2011)
    # gray, 0-255: noise against a blurred, noisier copy
    a = rng.uniform(0, 255, (192, 256))
    k = np.array([1.0, 2.0, 1.0]) / 4
    blur = np.apply_along_axis(lambda r: np.convolve(r, k, "same"), 1, np.apply_along_axis(lambda c: np.convolve(c, k, "same"), 0, a))
    write_case("noise_256x192", blur + rng.normal(0, 8, a.shape), a, 256, 192, "gray")
    # a gradient quantised to 16 levels (the original: its steps give every band content) against the smooth one
    yy, xx = np.mgrid[0:180, 0:200]
    grad = 40 + 150 * (xx / 199.0) * (0.6 + 0.4 * np.sin(yy / 30.0))
    write_case("gradient_200x180", grad, np.round(grad / 16) * 16, 200, 180, "gray")
    # the minimum size and odd sizes where every level rounds up
    m = rng.uniform(0, 255, (161, 161))
    write_case("min_161x161", np.clip(m + rng.normal(0, 20, m.shape), 0, 255), m, 161, 161, "gray")
    o = rng.uniform(0, 255, (163, 201))
    write_case("odd_201x163", np.clip(0.8 * o + 30 + rng.normal(0, 10, o.shape), 0, 255), o, 201, 163, "gray")
    # an identical pair
    same = rng.uniform(0, 255, (200, 176))
    write_case("identical_176x200", same, same, 176, 200, "gray")
    # evaluate layout: a non-square noisy pair (the [W, H] view), and inputs outside [0, 1]
    e = rng.random((176, 200, 3))
    write_case("evaluate_noise_200x176", np.clip(e + rng.normal(0, 0.2, e.shape), 0, 1), e, 200, 176, "evaluate")
    u1, u2 = rng.uniform(-2.0, 3.0, (170, 165, 3)), rng.uniform(-2.0, 3.0, (170, 165, 3))
    write_case("evaluate_outside_165x170", u1, 0.5 * (u1 + u2), 165, 170, "evaluate")
    # real renders: the shipped Pavillon networks at two thresholds
    lo, hi = pavillon_renders(192, 168, (0.1, 0.5))
    write_case("evaluate_pavillon_192x168", hi, lo, 192, 168, "evaluate",
               render="oracle, Pavillon K=16, image thr 0.5, reference thr 0.1")


if __name__ == "__main__":
    main()
