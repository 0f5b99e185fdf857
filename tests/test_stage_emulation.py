"""oracle/stage_emulation.py on the CPU: fma32 is a correctly rounded fp32 fma, the emulation restates the reference (the
oracle and the golden cases, at the tolerances the reference comparisons use), and deliberately wrong variants of it fail
the checks tests/test_stage_kernels_exact.py applies to the kernels (teeth)."""
from fractions import Fraction

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import adanerf_oracle as orc
from oracle import stage_emulation as se

F32 = np.float32
CASES = ["pav_k8_t0.2", "pav_k8_t0.5", "pav_k16_t0.15", "shaped_k8_t0.2", "rand_k8_t0.2", "ndc_k16_t0.15"]


# ------------------------------------------------------------------------------------------------------- fma32
def _round_f32(q):
    """Fraction -> the nearest fp32 (ties to even), gradual underflow included; exact arithmetic throughout."""
    if q == 0:
        return F32(0.0)
    sign, q = (-1 if q < 0 else 1), abs(q)
    e = q.numerator.bit_length() - q.denominator.bit_length()
    while Fraction(2) ** e > q:
        e -= 1
    while Fraction(2) ** (e + 1) <= q:
        e += 1
    ulp = Fraction(2) ** (max(e, -126) - 23)
    m = q / ulp
    n = m.numerator // m.denominator
    rem = m - n
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and n % 2 == 1):
        n += 1
    return F32(sign * float(n * ulp))


def _check_fma(a, b, c):
    a, b, c = (np.asarray(x, F32).ravel() for x in (a, b, c))
    got = se.fma32(a, b, c)
    want = np.array([_round_f32(Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z))) for x, y, z in zip(a, b, c)], F32)
    np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32))


def test_fma32_random_triples():
    rng = np.random.default_rng(0)
    n = 4000
    mant = lambda: rng.uniform(-2.0, 2.0, n)
    a = (mant() * 2.0 ** rng.integers(-30, 30, n)).astype(F32)
    b = (mant() * 2.0 ** rng.integers(-30, 30, n)).astype(F32)
    c = (mant() * 2.0 ** rng.integers(-70, 70, n)).astype(F32)
    _check_fma(a, b, c)
    # the operands posenc3's recurrence feeds it: fma(-2s, s, 1) with |s| <= 1
    s = rng.uniform(-1.0, 1.0, n).astype(F32)
    _check_fma(F32(-2) * s, s, np.ones(n, F32))


def test_fma32_adversarial_triples():
    """Products on an exact fp32 midpoint (1 + i 2^-12)(1 + j 2^-12), alone (ties to even), nudged by a c far below the
    last bit (round-to-odd must keep the direction), denormal c, and c cancelling the product's leading bits."""
    i = np.arange(1, 40, dtype=np.float64)
    a = np.repeat(1.0 + i * 2.0 ** -12, len(i)).astype(F32)
    b = np.tile(1.0 + i * 2.0 ** -12, len(i)).astype(F32)
    p_rn = (a.astype(np.float64) * b.astype(np.float64)).astype(F32)
    for c in (np.zeros_like(a), np.full_like(a, 2.0 ** -70), np.full_like(a, -2.0 ** -70), np.full_like(a, 2.0 ** -149),
              np.full_like(a, -3 * 2.0 ** -149), -p_rn, -np.nextafter(p_rn, F32(0)), np.full_like(a, -1.0), np.full_like(a, -0.5)):
        _check_fma(a, b, c)
        _check_fma(-a, b, c)
    # tiny products against a tiny / denormal addend
    t = np.array([2.0 ** -70, 3 * 2.0 ** -75, 2.0 ** -63 + 2.0 ** -86], F32)
    _check_fma(t, t, np.array([2.0 ** -149, -2.0 ** -140, 2.0 ** -126], F32))


# --------------------------------------------------------------------------------------- emulation == reference
@pytest.mark.parametrize("W,H", [(800, 800), (3, 801), (801, 799)])
def test_pixel_dir_is_the_reference_generator(W, H):
    fov = orc.SCENE_BARBERSHOP["fov"]
    ref = orc.generate_ray_directions(W, H, fov).reshape(-1, 3).astype(F32)
    np.testing.assert_array_equal(se.pixel_dir(W, H, fov), ref)
    np.testing.assert_array_equal(se.pixel_dir(W, H, fov, row0=H // 2, rows=2), ref[(H // 2) * W:(H // 2 + 2) * W])


@pytest.mark.parametrize("case", CASES)
def test_stage0_emulation_matches_the_reference(case):
    """Same bounds as test_gpu_parity's stage-0 checks against the reference's tensors."""
    g = load_golden(case)
    scene = g["meta"]["scene_params"]
    ro, rd, x0 = se.stage0(g["pose"], g["rot"], g["dirs"], scene)
    np.testing.assert_array_equal(rd, g["ray_d"])
    np.testing.assert_allclose(ro, g["ray_o"], rtol=0, atol=1e-6)
    if scene.get("use_ndc"):
        np.testing.assert_allclose(x0, g["x0"], rtol=0, atol=2e-5)
        return
    np.testing.assert_allclose(x0[:, :27], g["x0"][:, :27], rtol=0, atol=2e-6)
    err = np.abs(x0[:, 27:] - g["x0"][:, 27:])
    assert err.max() < 5e-4 and err[:, :3 + 6 * 4].max() < 2e-5, err.max()
    # and the torch oracle on a full-frame sample at a rotated pose
    dirs = orc.generate_ray_directions(800, 800, scene["fov"]).reshape(-1, 3).astype(F32)[::97]
    rot = orc.rotation_yaw(33.0)
    pose = torch.tensor(scene["view_cell_center"]) + torch.tensor([0.1, -0.05, 0.02])
    o_x0, o_ro, o_rd = orc.stage0_sphere_pos_dir(pose, rot, torch.from_numpy(dirs), scene)
    ro, rd, x0 = se.stage0(pose.numpy(), rot.numpy(), dirs, scene)
    np.testing.assert_array_equal(rd, o_rd.numpy())
    np.testing.assert_allclose(ro, o_ro.numpy(), rtol=0, atol=1e-6)
    assert np.abs(x0[:, :27] - o_x0.numpy()[:, :27]).max() < 2e-6
    assert np.abs(x0[:, 27:] - o_x0.numpy()[:, 27:]).max() < 5e-4


def _packed(g, K):
    z = g["z_nan"]
    mask = np.isfinite(z)
    return mask, np.repeat(np.arange(z.shape[0]), K).reshape(z.shape)[mask], z[mask]


@pytest.mark.parametrize("case", ["pav_k8_t0.2", "shaped_k8_t0.2", "ndc_k16_t0.15"])
def test_stage3_emulation_matches_the_reference(case):
    """Same bounds as test_gpu_parity's stage-3 checks (test_stage3_matches_reference, the NDC variant's stage 3)."""
    g = load_golden(case)
    scene = g["meta"]["scene_params"]
    mask, ray, z = _packed(g, g["meta"]["K"])
    x1 = se.stage3(scene, g["ray_o"], g["ray_d"], ray, z)
    ref = g["x1_nan"].reshape(-1, 90)[mask.flatten()]
    err = np.abs(x1 - ref)
    if scene.get("use_ndc"):
        assert np.abs(x1[:, :3] - ref[:, :3]).max() < 2e-5 * max(1.0, np.abs(ref[:, :3]).max())
        assert err[:, 63:].max() < 2e-5 and err[:, :63].max() < 5e-3, err.max()
    else:
        assert err[:, 63:].max() < 2e-6 and err[:, :3 + 6 * 4].max() < 2e-5 and err.max() < 5e-4, err.max()
    # the oracle on the same inputs
    zz = np.full(g["z_nan"].shape, np.inf, F32)
    zz[mask] = z
    o_x1, _, _ = orc.stage3_encode(torch.from_numpy(g["ray_o"]), torch.from_numpy(g["ray_d"]), torch.from_numpy(zz), scene)
    assert np.abs(x1[:, :3] - o_x1.numpy()[:, :3]).max() < 2e-5 * max(1.0, np.abs(x1[:, :3]).max())


def _sig32(logits):
    """fp32 sigmoid through float64 (within an ulp of the kernel's expf-based one)."""
    return (1.0 / (1.0 + np.exp(-np.asarray(logits, np.float64)))).astype(F32)


@pytest.mark.parametrize("case", ["pav_k8_t0.2", "pav_k16_t0.15", "shaped_k8_t0.2", "rand_k8_t0.2", "ndc_k16_t0.15"])
def test_stage5_emulation_matches_the_reference(case):
    """Both composites against the reference's rgb / weights at test_gpu_parity's 1e-6."""
    g = load_golden(case)
    m = g["meta"]
    K = m["K"]
    mask, _, z = _packed(g, K)
    cnt = mask.sum(1)
    off = np.concatenate([[0], np.cumsum(cnt)[:-1]])
    o2 = orc.stage2_sample(torch.from_numpy(g["raw0"]), m["thr"], K, m["scene_params"]["depth_range"],
                           no_depth_range=bool(m["scene_params"].get("use_ndc")))
    zp = o2["zp"].numpy()[mask]
    sig = _sig32(g["raw1_pad"].reshape(-1, 4)[mask.flatten()])
    for fn in (se.stage5_thread, se.stage5_warp):
        out = fn(sig, zp, z, off, cnt, K)
        np.testing.assert_allclose(out["rgb"], g["rgb"], rtol=0, atol=1e-6)
        np.testing.assert_allclose(out["weights"], g["weights"], rtol=0, atol=1e-6)


def test_stage5_emulation_matches_the_oracle_at_k128():
    rng = np.random.default_rng(9)
    n, K = 300, 128
    cnt = rng.integers(0, K + 1, n)
    off = np.cumsum(cnt) - cnt
    M = int(cnt.sum())
    raw1 = rng.standard_normal((M, 4)).astype(F32)
    zp, z = rng.uniform(0, 0.5, M).astype(F32), rng.uniform(0, 5, M).astype(F32)
    mapping = (np.arange(K)[None, :] < cnt[:, None]).flatten()
    zp_pad = np.zeros(n * K, F32)
    zp_pad[mapping] = zp
    ref = orc.stage5_composite(torch.from_numpy(raw1), torch.from_numpy(z), torch.from_numpy(zp_pad).view(n, K),
                               torch.from_numpy(mapping), n, K)
    out = se.stage5_warp(_sig32(raw1), zp, z, off, cnt, K)
    np.testing.assert_allclose(out["rgb"], ref["rgb"].numpy(), rtol=0, atol=2e-6)
    np.testing.assert_allclose(out["weights"], ref["weights"].numpy(), rtol=0, atol=2e-6)
    np.testing.assert_allclose(out["depth_map"], ref["depth_map"].numpy(), rtol=0, atol=2e-5)


# -------------------------------------------------------------------------------------------- posenc band bounds
def test_posenc_from_exact_anchors_is_within_the_band_bounds():
    """posenc3 from correctly rounded anchors stays inside the per-band bounds the kernel tests apply; the bound table is
    what the posenc.cuh comment quotes (1.7e-5 at bands 4 and 9; 3.8e-6 from correctly rounded anchors)."""
    bound = se.recurrence_band_bounds()
    assert bound.shape == (10,) and (np.diff(bound[:5]) > 0).all() and np.array_equal(bound[:5], bound[5:])
    assert 1.5e-5 < bound.max() < 1.7e-5, bound
    v = np.random.default_rng(1).uniform(-8, 8, (200000, 3)).astype(F32)
    err = np.abs(se.posenc3(v, 10) - se.posenc_f64(v, 10))[:, 3:].reshape(-1, 10, 2, 3).max(axis=(0, 2, 3))
    assert (err <= bound).all(), (err, bound)
    assert 3e-6 < err.max() < 4.5e-6, err


# ------------------------------------------------------------------------------------------------------ teeth
def test_teeth_no_band5_anchor():
    """Continuing the recurrence through band 5 breaks the per-band bound of the kernel test at bands >= 5."""
    v = np.random.default_rng(2).uniform(-8, 8, (50000, 3)).astype(F32)
    bad = se.posenc3(v, 10, anchor_every=10)
    err = np.abs(bad - se.posenc_f64(v, 10))[:, 3:].reshape(-1, 10, 2, 3).max(axis=(0, 2, 3))
    assert (err[5:] > se.recurrence_band_bounds()[5:]).all(), err
    # and the bit-for-bit recurrence check seeded with the correct anchors fails too
    good = se.posenc3(v, 10)
    assert not np.array_equal(se.posenc3(v, 10, anchors=good), bad)


@pytest.mark.parametrize("scene", [orc.SCENE_BARBERSHOP, orc.SCENE_PAVILLON_NDC])
def test_teeth_contracted_position(scene):
    """p = pose + nds t (stage 0) or o + d z (stage 3) contracted into an fma changes positions the kernel tests compare
    bit for bit."""
    dirs = se.pixel_dir(800, 800, scene["fov"])[::53]
    pose = np.asarray(scene["view_cell_center"], F32) + F32(0.3)
    rot = orc.rotation_yaw(20.0).numpy()
    ro, rd, x0 = se.stage0(pose, rot, dirs, scene)
    ro_c, _, x0_c = se.stage0(pose, rot, dirs, scene, contract=True)
    assert not np.array_equal(ro, ro_c) and not np.array_equal(x0, x0_c)
    n = ro.shape[0]
    ray = np.repeat(np.arange(n), 4)
    z = np.random.default_rng(3).uniform(0.01, 6.0, 4 * n).astype(F32)
    pos, _ = se.sample_inputs(scene, ro, rd, ray, z)
    pos_c, _ = se.sample_inputs(scene, ro, rd, ray, z, contract=True)
    assert not np.array_equal(pos, pos_c)


def _exact_sigmoid_inputs(K, n_per=40, seed=4):
    """Stage-5 inputs whose sigmoids are exact (logits -200 / 0 / 200 -> 0, 1/2, 1) with zp, z arbitrary fp32 values."""
    rng = np.random.default_rng(seed)
    edges = [c for c in (0, 1, 2, 31, 32, 33, 63, 64, 65, 95, 96, 97, 127, 128, K - 1, K) if 0 <= c <= K]
    cnt = np.concatenate([np.repeat(edges, 3), rng.integers(0, K + 1, n_per)])
    off = np.cumsum(cnt) - cnt
    M = int(cnt.sum())
    logits = rng.choice(np.array([-200.0, 0.0, 200.0], F32), (M, 4))
    zp = rng.choice(np.array([0.0, 1.0, 2.0, -0.75, 0.5, 1.5], F32), M)
    zp = np.where(rng.random(M) < 0.5, zp, rng.uniform(-0.5, 1.5, M).astype(F32))
    z = (rng.standard_normal(M) * 4).astype(F32)
    return logits, zp, z, off, cnt


@pytest.mark.parametrize("K", [16, 100])
def test_teeth_transmittance_without_eps(K):
    logits, zp, z, off, cnt = _exact_sigmoid_inputs(K)
    sig = _sig32(logits)
    assert set(np.unique(sig)) <= {F32(0), F32(0.5), F32(1)}
    fn = se.stage5_warp if K > 32 else se.stage5_thread
    good, bad = fn(sig, zp, z, off, cnt, K), fn(sig, zp, z, off, cnt, K, eps=F32(0))
    assert not np.array_equal(good["weights"], bad["weights"]) and not np.array_equal(good["rgb"], bad["rgb"])


def test_teeth_sequential_product_in_the_warp_composite():
    logits, zp, z, off, cnt = _exact_sigmoid_inputs(100)
    sig = _sig32(logits)
    good = se.stage5_warp(sig, zp, z, off, cnt, 100)
    bad = se.stage5_warp(sig, zp, z, off, cnt, 100, tree=False)
    assert not np.array_equal(good["weights"], bad["weights"])
    # the thread kernel's chain is not the warp kernel's either: the two emulations are not interchangeable
    assert not np.array_equal(good["weights"], se.stage5_thread(sig, zp, z, off, cnt, 100)["weights"])
