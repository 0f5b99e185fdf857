"""FLIP without a GPU: the torch emulation (oracle/flip_emulation.py) against the reference's own fp32 maps
(tests/golden/flip_*, written by oracle/gen_flip_golden.py from the unmodified util/flip_loss.py), and the build side of
adn_image_flip: the exported symbol, the header, and SASS of the FLIP kernels for sm_90a."""
import ctypes
import glob
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT, load_golden
from oracle import flip_emulation as fe

CASES = sorted({os.path.basename(p).split(".")[0] for p in glob.glob(os.path.join(GOLDEN, "flip_*"))})


def tolerance(g):
    """Per pixel: above the reference's own fp32-vs-fp64 spread for the case, with a floor."""
    return max(1e-4, 4 * float(g["spread"]))


def check_against_golden(got_map, got_mean, g, what):
    want = g["map"].astype(np.float64)
    got = np.asarray(got_map, np.float64).reshape(want.shape)
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan), f"{what}: NaN masks differ"
    err = np.abs(got[~nan] - want[~nan]).max() if (~nan).any() else 0.0
    assert err <= tolerance(g), f"{what}: max |map - reference| = {err:.3g} > {tolerance(g):.3g}"
    ref_mean = float(g["mean"])
    if np.isnan(ref_mean):
        assert np.isnan(got_mean), what
    else:
        # 1e-6 relative, or above the reference's own fp32-vs-fp64 difference of the mean where a few pixels make it up
        tol = max(1e-6 * abs(ref_mean), 4 * abs(ref_mean - g["meta"]["mean_fp64"]))
        assert abs(got_mean - ref_mean) <= tol, f"{what}: mean {got_mean!r} vs {ref_mean!r}"


def test_golden_cases_cover_the_documented_set():
    names = set(CASES)
    for want in ("flip_noise_256x192", "flip_smooth_160x120", "flip_pattern_64x64", "flip_outside_48x40", "flip_nan_32x32",
                 "flip_identical_40x24", "flip_tiny_7x5", "flip_tiny_1x1", "flip_ppd30_64x48", "flip_ppdcap_64x48",
                 "flip_pavillon_48x40"):
        assert want in names


@pytest.mark.parametrize("case", CASES)
def test_emulation_matches_reference(case):
    g = load_golden(case)
    m = g["meta"]
    W, H, ppd = m["W"], m["H"], m["ppd"]
    assert (fe.csf_radius(ppd), fe.feature_radius(ppd)) == (m["radius_csf"], m["radius_feature"])
    assert abs(fe.cmax() - m["cmax"]) <= 1e-12 * m["cmax"]
    img, ref = torch.from_numpy(g["image"]), torch.from_numpy(g["reference"])
    fmap, mean = fe.flip(img, ref, W, H, ppd)
    check_against_golden(fmap.numpy(), mean, g, case)
    # evaluate.py passes (test, reference) into compute_flip(reference, test): the metric is symmetric
    fmap2, _ = fe.flip(ref, img, W, H, ppd)
    assert torch.equal(fmap.isnan(), fmap2.isnan())
    ok = ~fmap.isnan()
    assert (fmap[ok] - fmap2[ok]).abs().max().item() <= 1e-12 if ok.any() else True


def test_identical_pair_is_exactly_zero():
    g = load_golden("flip_identical_40x24")
    assert not g["map"].any() and float(g["mean"]) == 0.0
    img = torch.from_numpy(g["image"])
    fmap, mean = fe.flip(img, img.clone(), 40, 24)
    assert not fmap.any() and mean == 0.0


def test_nan_pixel_spreads_over_the_csf_radius():
    g = load_golden("flip_nan_32x32")
    nan = np.isnan(g["map"])
    r = g["meta"]["radius_csf"]
    block = np.zeros_like(nan)
    block[max(0, 5 - r):5 + r + 1, max(0, 5 - r):5 + r + 1] = True
    assert r == 10 and np.array_equal(nan, block)


def test_default_ppd_is_evaluate_py():
    from adanerf_b200.renderer import EVALUATE_PPD
    assert EVALUATE_PPD == fe.EVALUATE_PPD
    assert abs(EVALUATE_PPD - 67.0206) < 1e-4
    assert (fe.csf_radius(EVALUATE_PPD), fe.feature_radius(EVALUATE_PPD)) == (10, 9)
    assert fe.csf_radius(200.0) == 28      # the cap: the kernels stage radii up to 28


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as g
    g.build()
    return g


def test_symbol_is_declared_exported_and_listed(built):
    lib = ctypes.CDLL(built.LIB)
    assert hasattr(lib, "adn_image_flip")
    from adanerf_b200._lib import SYMBOLS
    assert "adn_image_flip" in SYMBOLS
    assert "flip.cu" in built.SOURCES and "flip.cuh" in built.HEADERS
    with open(os.path.join(ROOT, "include", "adanerf_b200.h")) as f:
        decl = re.search(r"adn_status adn_image_flip\(([^)]*)\)", f.read())
    assert decl and "stream" not in decl.group(1)


def test_flip_kernels_are_sm90a_simt(built):
    cuobjdump = os.path.join(built.CUDA_HOME, "bin", "cuobjdump")
    r = subprocess.run([cuobjdump, "-sass", built.LIB], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    funcs = re.split(r"\n\s*Function : ", r.stdout)
    flip = {f.split("\n", 1)[0].strip(): f for f in funcs if "flip_" in f.split("\n", 1)[0]}
    for name in ("flip_rows_kernel", "flip_cols_kernel", "flip_sum_kernel"):
        hits = [k for k in flip if name in k]
        assert hits, f"{name} not in the library's SASS"
        assert "HMMA" not in flip[hits[0]]
    assert "arch = sm_90a" in r.stdout
