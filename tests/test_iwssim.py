"""IW-SSIM without a GPU: the restated Laplacian pyramid (oracle/laplacian_pyramid.py), the torch emulation
(oracle/iwssim_emulation.py) against the reference's own scores (tests/golden/iwssim_*, written by
oracle/gen_iwssim_golden.py from the unmodified util/IW_SSIM_PyTorch.py), the evaluate-layout conversion bit for bit, the
Python wrapper's argument checks, and the build side of adn_image_iwssim: the exported symbol, the header and the SASS of
its kernels for sm_90a."""
import ctypes
import glob
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT, load_golden
from oracle import iwssim_emulation as ie
from oracle import laplacian_pyramid as lp

CASES = sorted({os.path.basename(p).split(".")[0] for p in glob.glob(os.path.join(GOLDEN, "iwssim_*"))})


def tolerance(ref32, ref64):
    """What a device result may differ from the reference's fp64 result by: the reference's own fp32-vs-fp64 spread, with
    a floor of 2e-6."""
    return max(abs(ref32 - ref64), 2e-6)


def test_golden_cases_cover_the_documented_set():
    for want in ("iwssim_noise_256x192", "iwssim_gradient_200x180", "iwssim_min_161x161", "iwssim_odd_201x163",
                 "iwssim_identical_176x200", "iwssim_evaluate_noise_200x176", "iwssim_evaluate_outside_165x170",
                 "iwssim_evaluate_pavillon_192x168"):
        assert want in CASES
    for case in CASES:
        m = load_golden(case)["meta"]
        assert np.isfinite(m["score_fp32"]) and np.isfinite(m["score_fp64"]), case


@pytest.mark.parametrize("shape", [(161, 161), (163, 201), (200, 176), (256, 192)])
def test_pyramid_reconstructs_its_input(shape):
    x = np.random.default_rng(shape[0] * shape[1]).uniform(0, 255, shape)
    bands = lp.laplacian_pyramid(x, 5)
    assert [b.shape for b in bands] == [(-(-shape[0] // 2 ** l), -(-shape[1] // 2 ** l)) for l in range(5)]
    assert np.abs(lp.reconstruct(bands) - x).max() <= 1e-12 * np.abs(x).max()


@pytest.mark.parametrize("c", [1.0, -3.5, 255.0])
def test_constant_image_has_zero_bands(c):
    bands = lp.laplacian_pyramid(np.full((163, 201), c), 5)
    for b in bands[:-1]:
        assert np.abs(b).max() <= 1e-12 * abs(c)
    assert np.abs(bands[-1] - 16 * c).max() <= 1e-12 * abs(c)


@pytest.mark.parametrize("case", CASES)
def test_emulation_matches_reference_fp64(case):
    g = load_golden(case)
    m = g["meta"]
    out = ie.iwssim(torch.from_numpy(g["original"]), torch.from_numpy(g["distorted"]), torch.float64)
    assert abs(out["score"] - m["score_fp64"]) <= 1e-10, (out["score"], m["score_fp64"])
    assert np.abs(np.array(out["wmcs"]) - np.array(m["wmcs_fp64"])).max() <= 1e-10
    assert out["score"] == float(g["score_emulation"])
    # the device is held to the reference's own fp32-vs-fp64 spread; it must be below 1e-3 for that to mean anything
    assert tolerance(m["score_fp32"], m["score_fp64"]) < 1e-3


@pytest.mark.parametrize("case", CASES)
def test_metric_images_match_fixture_bit_for_bit(case):
    g = load_golden(case)
    m = g["meta"]
    o, d = ie.metric_images(torch.from_numpy(g["image"]), torch.from_numpy(g["reference"]), m["W"], m["H"], m["layout"])
    assert torch.equal(o.view(torch.int32), torch.from_numpy(g["original"]).view(torch.int32))
    assert torch.equal(d.view(torch.int32), torch.from_numpy(g["distorted"]).view(torch.int32))
    if m["layout"] == "evaluate":
        assert o.shape == (m["W"], m["H"])                 # rgb2gray(x.view(W, H, -1)): W rows of H pixels
        assert set(np.unique(g["original"]).tolist()) <= set(range(-3, 5))


def test_identical_pair_scores_one():
    g = load_golden("iwssim_identical_176x200")
    assert abs(g["meta"]["score_fp64"] - 1.0) <= 1e-12 and abs(float(g["score_emulation"]) - 1.0) <= 1e-12


def test_scale_weights_are_the_references_fp32_values():
    assert ie.WEIGHTS[0] == float(np.float32(0.0448)) and ie.WEIGHTS[0] != 0.0448
    assert abs(sum(ie.WEIGHTS) - 1.0001) < 1e-6


def test_wrapper_checks_arguments_without_a_device():
    from adanerf_b200.renderer import IWSSIM_MIN_SIZE, Renderer
    r = Renderer.__new__(Renderer)           # argument checks run before the wrapper touches the library or a device
    W, H = 200, 170
    rgb, gray = torch.zeros((H * W, 3)), torch.zeros(H * W)
    bad = [
        (rgb, rgb, W, H, "rgb"),                                    # unknown layout
        (rgb, rgb, IWSSIM_MIN_SIZE - 1, H, "evaluate"),             # too small
        (rgb, rgb, W, IWSSIM_MIN_SIZE - 1, "evaluate"),
        (gray, gray, W, H, "evaluate"),                             # gray planes in the evaluate layout
        (rgb, rgb, W, H, "gray"),                                   # RGB in the gray layout
        (rgb, rgb[:-1], W, H, "evaluate"),
        (rgb, rgb, H, W + 1, "evaluate"),
        (rgb.reshape(W, H, 3), rgb.reshape(W, H, 3), W, H, "evaluate"),   # [W, H, 3] is not a frame of W x H
        (gray.reshape(H, W), gray, W, H, "gray"),                   # shapes differ
    ]
    for img, ref, w, h, layout in bad:
        with pytest.raises(ValueError):
            r.iw_ssim(img, ref, w, h, layout=layout)


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as g
    g.build()
    return g


def test_symbol_is_declared_exported_and_listed(built):
    lib = ctypes.CDLL(built.LIB)
    assert hasattr(lib, "adn_image_iwssim")
    from adanerf_b200._lib import SYMBOLS
    assert "adn_image_iwssim" in SYMBOLS
    assert "iwssim.cu" in built.SOURCES and "iwssim.cuh" in built.HEADERS
    with open(os.path.join(ROOT, "include", "adanerf_b200.h")) as f:
        h = f.read()
    decl = re.search(r"adn_status adn_image_iwssim\(([^)]*)\)", h)
    assert decl and "stream" not in decl.group(1)
    assert re.search(r"#define ADN_IWSSIM_GRAY\s+0", h) and re.search(r"#define ADN_IWSSIM_EVALUATE_RGB\s+1", h)


def test_iwssim_kernels_are_sm90a_simt(built):
    cuobjdump = os.path.join(built.CUDA_HOME, "bin", "cuobjdump")
    r = subprocess.run([cuobjdump, "-sass", built.LIB], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    funcs = re.split(r"\n\s*Function : ", r.stdout)
    iw = {f.split("\n", 1)[0].strip(): f for f in funcs if "iwssim_" in f.split("\n", 1)[0]}
    for name in ("iwssim_gray_kernel", "iwssim_down_kernel", "iwssim_band_kernel", "iwssim_cov_kernel",
                 "iwssim_eig_kernel", "iwssim_main_kernel", "iwssim_final_kernel"):
        hits = [k for k in iw if name in k]
        assert hits, f"{name} not in the library's SASS"
        assert "HMMA" not in iw[hits[0]]
    assert "DFMA" in iw[[k for k in iw if "iwssim_main_kernel" in k][0]]     # the statistics run in fp64
    assert "arch = sm_90a" in r.stdout
