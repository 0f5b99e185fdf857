"""IW-SSIM on the H100 (adn_image_iwssim, Renderer.iw_ssim): the device score and wmcs against the reference's fp64 results
(tests/golden/iwssim_*), within the reference's own fp32-vs-fp64 spread or 2e-6, whichever is larger; full-frame Pavillon
renders against the fp64 torch emulation on the device; identical inputs, repeated calls, order behind a render on another
stream, NaN for a scale that cannot be inverted, every refused argument with nothing launched, and the wrapper's errors."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import adanerf_oracle as orc
from oracle import iwssim_emulation as ie
from test_iwssim import CASES, tolerance

pytestmark = pytest.mark.gpu

ADN_ERR_INVALID = 1
LAYOUT = {"gray": 0, "evaluate": 1}
RX = torch.tensor([[1, 0, 0], [0, 0, -1], [0, 1, 0]], dtype=torch.float32)   # camera -z -> world +y


@pytest.fixture(scope="module")
def renderer(pavillon_weights):
    import __graft_entry__ as g
    g.build()
    from adanerf_b200 import Renderer
    sd0, sd1 = pavillon_weights
    r = Renderer(orc.SCENE_PAVILLON, device=0, sampling_net=sd0, shading_net=sd1)
    yield r
    r.close()


def _launches(r):
    return r.stats()["kernel_launches"]


def _check(out, score64, wmcs64, tol, what):
    err = [abs(a - b) for a, b in zip(out["scales"], wmcs64)]
    assert max(err) <= tol, f"{what}: wmcs {out['scales']} vs fp64 {wmcs64} (tolerance {tol:.3g})"
    assert abs(out["score"] - score64) <= tol, f"{what}: score {out['score']!r} vs fp64 {score64!r} (tolerance {tol:.3g})"


@pytest.mark.parametrize("case", CASES)
def test_device_matches_reference(renderer, case):
    g = load_golden(case)
    m = g["meta"]
    img, ref = torch.from_numpy(g["image"]).cuda(), torch.from_numpy(g["reference"]).cuda()
    out = renderer.iw_ssim(img, ref, m["W"], m["H"], layout=m["layout"])
    _check(out, m["score_fp64"], m["wmcs_fp64"], tolerance(m["score_fp32"], m["score_fp64"]), case)
    again = renderer.iw_ssim(img, ref, m["W"], m["H"], layout=m["layout"])
    assert again == out                                       # the same bits


def _render(r, W, H, thr, K=16):
    pose = torch.tensor(orc.SCENE_PAVILLON["view_cell_center"]) + torch.tensor([0.05, -0.03, 0.02])
    return r.render_camera(pose, RX, W, H, thr, K)["rgb"]


@pytest.mark.parametrize("W,H", [(800, 800), (1600, 1600), (960, 544)])
def test_pavillon_renders_match_fp64_emulation(renderer, W, H):
    """Evaluate layout on whole renders, and the same renders' gray planes on the 0-255 scale (where the bands are not
    0s and 1s): the device against the fp64 emulation, within the emulation's own fp32-vs-fp64 spread or 2e-6."""
    a, b = _render(renderer, W, H, 0.5), _render(renderer, W, H, 0.1)
    torch.cuda.synchronize()
    for layout in ("evaluate", "gray"):
        if layout == "gray":
            a = (255 * (0.2989 * a[:, 0] + 0.5870 * a[:, 1] + 0.1140 * a[:, 2])).contiguous()
            b = (255 * (0.2989 * b[:, 0] + 0.5870 * b[:, 1] + 0.1140 * b[:, 2])).contiguous()
        out = renderer.iw_ssim(a, b, W, H, layout=layout)
        o, d = ie.metric_images(a, b, W, H, layout)
        e64 = ie.iwssim(o, d, torch.float64, device="cuda")
        e32 = ie.iwssim(o, d, torch.float32, device="cuda")
        tol = max(tolerance(e32["score"], e64["score"]), max(abs(x - y) for x, y in zip(e32["wmcs"], e64["wmcs"])))
        _check(out, e64["score"], e64["wmcs"], tol, f"{W}x{H} {layout}")
        assert 0.0 < out["score"] <= 1.0 + 1e-6


def test_identical_inputs_score_one(renderer):
    W, H = 401, 263
    x = _render(renderer, W, H, 0.3)
    torch.cuda.synchronize()
    out = renderer.iw_ssim(x, x.clone(), W, H)
    assert abs(out["score"] - 1.0) <= 1e-6 and all(abs(s - 1.0) <= 1e-6 for s in out["scales"])
    gray = torch.rand(H * W, device="cuda") * 255
    out = renderer.iw_ssim(gray, gray.clone(), W, H, layout="gray")
    assert abs(out["score"] - 1.0) <= 1e-6


def test_call_after_a_render_on_a_side_stream(renderer):
    W = H = 400
    ref = _render(renderer, W, H, 0.05)
    torch.cuda.synchronize()
    img = _render(renderer, W, H, 0.3)
    torch.cuda.synchronize()
    want = renderer.iw_ssim(img, ref, W, H)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        img2 = _render(renderer, W, H, 0.3)
        got = renderer.iw_ssim(img2, ref, W, H)                     # no synchronisation in between
    torch.cuda.synchronize()
    assert got == want


def _raw(r, a, b, W, H, layout):
    score, scales = C.c_double(), (C.c_double * 5)()
    st = r.lib.adn_image_iwssim(r.handle, a.data_ptr(), b.data_ptr(), W, H, layout, C.byref(score), scales)
    return st, score.value, list(scales)


def test_uninvertible_scales_give_nan(renderer):
    W, H = 200, 176
    gen = torch.Generator(device="cuda").manual_seed(5)
    img = torch.rand((H * W,), device="cuda", generator=gen) * 255
    # an all-zero reference: every band of the original is 0, so is its covariance
    st, score, scales = _raw(renderer, img, torch.zeros_like(img), W, H, LAYOUT["gray"])
    assert st == 0 and math.isnan(score) and all(math.isnan(s) for s in scales[:4])
    # one NaN pixel in either image
    for which in (0, 1):
        a, b = img.clone(), (img + 10 * torch.rand(img.shape, device="cuda", generator=gen)).contiguous()
        (a if which == 0 else b)[H // 2 * W + W // 3] = float("nan")
        st, score, _ = _raw(renderer, a, b, W, H, LAYOUT["gray"])
        assert st == 0 and math.isnan(score), which
    # and the call after them is unaffected
    st, score, _ = _raw(renderer, img, img.clone(), W, H, LAYOUT["gray"])
    assert st == 0 and abs(score - 1.0) <= 1e-6


def test_invalid_arguments_launch_nothing(renderer):
    r = renderer
    lib = r.lib
    W, H = 170, 161
    a = torch.rand((H * W, 3), device="cuda")
    b = torch.rand((H * W, 3), device="cuda")
    score, scales = C.c_double(), (C.c_double * 5)()
    good = (a.data_ptr(), b.data_ptr(), W, H, 1, C.byref(score), scales)
    assert lib.adn_image_iwssim(r.handle, *good) == 0
    bad = [
        (None, b.data_ptr(), W, H, 1, C.byref(score), scales),
        (a.data_ptr(), None, W, H, 1, C.byref(score), scales),
        (a.data_ptr(), b.data_ptr(), W, H, 1, None, scales),
        (a.data_ptr(), b.data_ptr(), 160, H, 1, C.byref(score), scales),
        (a.data_ptr(), b.data_ptr(), W, 160, 1, C.byref(score), scales),
        (a.data_ptr(), b.data_ptr(), 0, H, 1, C.byref(score), scales),
        (a.data_ptr(), b.data_ptr(), -W, H, 1, C.byref(score), scales),
        (a.data_ptr(), b.data_ptr(), 65536, 32768, 1, C.byref(score), scales),   # W * H = 2^31
        (a.data_ptr(), b.data_ptr(), W, H, 2, C.byref(score), scales),
        (a.data_ptr(), b.data_ptr(), W, H, -1, C.byref(score), scales),
    ]
    for args in bad:
        n0 = _launches(r)
        assert lib.adn_image_iwssim(r.handle, *args) == ADN_ERR_INVALID, args
        assert _launches(r) == n0, args
    assert lib.adn_image_iwssim(None, *good) == ADN_ERR_INVALID
    # scale_out may be NULL; the gray layout reads [H*W] planes
    n0 = _launches(r)
    assert lib.adn_image_iwssim(r.handle, a.data_ptr(), b.data_ptr(), W, H, 1, C.byref(score), None) == 0
    ga, gb = a[:, 0].contiguous(), b[:, 0].contiguous()
    assert lib.adn_image_iwssim(r.handle, ga.data_ptr(), gb.data_ptr(), W, H, 0, C.byref(score), scales) == 0
    assert _launches(r) - n0 == 20
    assert np.isfinite(score.value)


def test_wrapper_errors_and_graph_capture(renderer):
    from adanerf_b200 import AdnError
    r = renderer
    W, H = 170, 161
    a = torch.rand((H * W, 3), device="cuda")
    for img, ref, w, h, layout in [(a, a[:-1], W, H, "evaluate"), (a, a, W + 1, H, "evaluate"), (a, a, W, H, "gray"),
                                   (a.reshape(-1), a.reshape(-1), W, H, "evaluate"), (a, a, W, H, "lab"),
                                   (a, a, 160, H, "evaluate")]:
        with pytest.raises(ValueError):
            r.iw_ssim(img, ref, w, h, layout=layout)
    out = r.iw_ssim(a.reshape(H, W, 3), a.reshape(H, W, 3), W, H)
    assert len(out["scales"]) == 5 and abs(out["score"] - 1.0) <= 1e-6
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    err = None
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        try:
            r.iw_ssim(a, a, W, H)
        except AdnError as e:
            err = e
    del g
    assert err is not None and err.status == ADN_ERR_INVALID and "capturing a CUDA graph" in str(err)
    assert abs(r.iw_ssim(a, a, W, H)["score"] - 1.0) <= 1e-6
