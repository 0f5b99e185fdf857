"""FLIP on the H100 (adn_image_flip, Renderer.flip): the device map and mean against the reference's own fp32 maps
(tests/golden/flip_*), against the fp64 torch emulation on the device at odd sizes and on full-frame Pavillon renders;
exact zeros for identical inputs, bit-identical results for swapped arguments and repeated calls; order behind a render on
another stream; every refused argument, with nothing launched."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import adanerf_oracle as orc
from oracle import flip_emulation as fe
from test_flip import CASES, check_against_golden

pytestmark = pytest.mark.gpu

ADN_ERR_INVALID = 1
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


def _bits(t):
    return t.detach().cpu().contiguous().view(torch.int32)


def _launches(r):
    return r.stats()["kernel_launches"]


@pytest.mark.parametrize("case", CASES)
def test_device_matches_reference(renderer, case):
    g = load_golden(case)
    m = g["meta"]
    img, ref = torch.from_numpy(g["image"]).cuda(), torch.from_numpy(g["reference"]).cuda()
    out = renderer.flip(img, ref, m["W"], m["H"], m["ppd"])
    assert out["map"].shape == (m["H"], m["W"])
    check_against_golden(out["map"].cpu().numpy(), out["mean"], g, case)
    # swapped arguments and a second call: the same bits
    again = renderer.flip(ref, img, m["W"], m["H"], m["ppd"])
    assert torch.equal(_bits(again["map"]), _bits(out["map"]))
    assert math.isnan(out["mean"]) and math.isnan(again["mean"]) or again["mean"] == out["mean"]
    twice = renderer.flip(img, ref, m["W"], m["H"], m["ppd"])
    assert torch.equal(_bits(twice["map"]), _bits(out["map"]))
    assert math.isnan(out["mean"]) or twice["mean"] == out["mean"]


def test_identical_inputs_give_exact_zeros(renderer):
    img = torch.rand((799 * 801, 3), device="cuda")
    out = renderer.flip(img, img.clone(), 801, 799)
    assert not out["map"].any() and out["mean"] == 0.0


def _against_fp64(renderer, img, ref, W, H, ppd=fe.EVALUATE_PPD):
    """The device result against the fp64 emulation, within 4x the emulation's own fp32-vs-fp64 spread (floor 1e-4 per
    pixel, 1e-6 relative on the mean)."""
    out = renderer.flip(img, ref, W, H, ppd)
    m64, mean64 = fe.flip(img, ref, W, H, ppd, torch.float64)
    m32, mean32 = fe.flip(img, ref, W, H, ppd, torch.float32)
    ok = ~m64.isnan()
    assert torch.equal(out["map"].isnan(), ~ok)
    spread = (m32[ok].double() - m64[ok]).abs().max().item() if ok.any() else 0.0
    err = (out["map"][ok].double() - m64[ok]).abs().max().item() if ok.any() else 0.0
    assert err <= max(1e-4, 4 * spread), f"{W}x{H}: max |map - fp64| = {err:.3g} (fp32 emulation: {spread:.3g})"
    tol = max(1e-6 * abs(mean64), 4 * abs(mean32 - mean64))
    assert abs(out["mean"] - mean64) <= tol, f"{W}x{H}: mean {out['mean']!r} vs fp64 {mean64!r}"
    return out


@pytest.mark.parametrize("W,H", [(801, 799), (33, 17), (1, 1000), (1000, 1)])
def test_odd_sizes_match_fp64_emulation(renderer, W, H):
    gen = torch.Generator(device="cuda").manual_seed(W * 7919 + H)
    img = torch.rand((H * W, 3), device="cuda", generator=gen)
    ref = (img + 0.1 * torch.randn((H * W, 3), device="cuda", generator=gen)).clamp(0, 1)
    _against_fp64(renderer, img, ref, W, H)
    _against_fp64(renderer, img.reshape(H, W, 3), ref.reshape(H, W, 3), W, H, ppd=30.0)   # [H, W, 3] input, another ppd


def _render(r, W, H, thr, K=16):
    pose = torch.tensor(orc.SCENE_PAVILLON["view_cell_center"]) + torch.tensor([0.05, -0.03, 0.02])
    return r.render_camera(pose, RX, W, H, thr, K)["rgb"]


@pytest.mark.parametrize("size", [800, 1600])
def test_pavillon_renders_match_fp64_emulation(renderer, size):
    a, b = _render(renderer, size, size, 0.5), _render(renderer, size, size, 0.1)
    torch.cuda.synchronize()
    out = _against_fp64(renderer, a, b, size, size)
    assert 0.0 < out["mean"] < 1.0


def test_flip_after_a_render_on_a_side_stream(renderer):
    W = H = 400
    ref = _render(renderer, W, H, 0.05)
    torch.cuda.synchronize()
    img = _render(renderer, W, H, 0.3)
    torch.cuda.synchronize()
    want = renderer.flip(img, ref, W, H)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        img2 = _render(renderer, W, H, 0.3)
        got = renderer.flip(img2, ref, W, H)                           # no synchronisation in between
    torch.cuda.synchronize()
    assert torch.equal(_bits(got["map"]), _bits(want["map"])) and got["mean"] == want["mean"]


def test_invalid_arguments_launch_nothing(renderer):
    r = renderer
    lib = r.lib
    W, H = 16, 8
    a = torch.rand((H * W, 3), device="cuda")
    b = torch.rand((H * W, 3), device="cuda")
    fmap = torch.empty((H, W), device="cuda")
    mean = C.c_double()
    good = (a.data_ptr(), b.data_ptr(), W, H, fe.EVALUATE_PPD, fmap.data_ptr(), C.byref(mean))
    assert lib.adn_image_flip(r.handle, *good) == 0
    bad = [
        (None, b.data_ptr(), W, H, fe.EVALUATE_PPD, fmap.data_ptr(), C.byref(mean)),
        (a.data_ptr(), None, W, H, fe.EVALUATE_PPD, fmap.data_ptr(), C.byref(mean)),
        (a.data_ptr(), b.data_ptr(), W, H, fe.EVALUATE_PPD, None, None),
        (a.data_ptr(), b.data_ptr(), 0, H, fe.EVALUATE_PPD, fmap.data_ptr(), C.byref(mean)),
        (a.data_ptr(), b.data_ptr(), W, 0, fe.EVALUATE_PPD, fmap.data_ptr(), C.byref(mean)),
        (a.data_ptr(), b.data_ptr(), -3, H, fe.EVALUATE_PPD, fmap.data_ptr(), C.byref(mean)),
        (a.data_ptr(), b.data_ptr(), 65536, 65536, fe.EVALUATE_PPD, fmap.data_ptr(), C.byref(mean)),   # W * H >= 2^31
        (a.data_ptr(), b.data_ptr(), W, H, float("nan"), fmap.data_ptr(), C.byref(mean)),
        (a.data_ptr(), b.data_ptr(), W, H, float("inf"), fmap.data_ptr(), C.byref(mean)),
        (a.data_ptr(), b.data_ptr(), W, H, 0.0, fmap.data_ptr(), C.byref(mean)),
        (a.data_ptr(), b.data_ptr(), W, H, -67.0, fmap.data_ptr(), C.byref(mean)),
        (a.data_ptr(), b.data_ptr(), W, H, 200.0001, fmap.data_ptr(), C.byref(mean)),
    ]
    for args in bad:
        n0 = _launches(r)
        assert lib.adn_image_flip(r.handle, *args) == ADN_ERR_INVALID, args
        assert _launches(r) == n0, args
    assert lib.adn_image_flip(None, *good) == ADN_ERR_INVALID
    # the cap itself, only the mean, only the map
    n0 = _launches(r)
    assert lib.adn_image_flip(r.handle, a.data_ptr(), b.data_ptr(), W, H, 200.0, None, C.byref(mean)) == 0
    assert lib.adn_image_flip(r.handle, a.data_ptr(), b.data_ptr(), W, H, 200.0, fmap.data_ptr(), None) == 0
    assert _launches(r) - n0 == 6
    assert torch.isfinite(fmap).all()


def test_wrapper_shape_errors_and_graph_capture(renderer):
    from adanerf_b200 import AdnError
    r = renderer
    W, H = 16, 8
    a = torch.rand((H * W, 3), device="cuda")
    for img, ref, w, h in [(a, a[:-1], W, H), (a, a, H, W + 1), (a.reshape(-1), a.reshape(-1), W, H),
                           (a.reshape(H, W, 3), a, W, H), (a.reshape(W, H, 3), a.reshape(W, H, 3), W, H), (a, a, 0, H)]:
        with pytest.raises(ValueError):
            r.flip(img, ref, w, h)
    assert r.flip(a.reshape(H, W, 3), a.reshape(H, W, 3), W, H, want_map=False)["map"] is None
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    err = None
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        try:
            r.flip(a, a, W, H)
        except AdnError as e:
            err = e
    del g
    assert err is not None and err.status == ADN_ERR_INVALID and "capturing a CUDA graph" in str(err)
    assert r.flip(a, a, W, H)["mean"] == 0.0
