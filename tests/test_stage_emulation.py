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


# ------------------------------------------------------------------------------------------------- depth tables
LOG_SCENES = {"barbershop": orc.SCENE_BARBERSHOP, "pavillon": orc.SCENE_PAVILLON}


def _world64(z, scene):
    """LogTransform.to_world in float64 on the fp32 scene fields and the exact fp32 z; also returns w = the power."""
    dr0, dr1 = float(F32(scene["depth_range"][0])), float(F32(scene["depth_range"][1]))
    w = (dr1 - dr0 + 1.0) ** np.asarray(z, F32).astype(np.float64)
    return (w - 1.0) + dr0, w


def _dense_z(K):
    t = se.linspace01(K)[:K] + F32(0.5 / K)
    return F32(0.001) * (F32(1) - t) + F32(1.0) * t


@pytest.mark.parametrize("name", sorted(LOG_SCENES))
def test_depth_tables_within_an_ulp_of_float64(name):
    """Both tables are within 1 ulp of the power w = (max_v + 1)^z of the float64 formula: pow is correctly rounded (up to
    glibc's < 1 ulp), (w - 1) and + dr0 add one rounding each.  Relative to the table value itself the error is larger where
    (w - 1) + dr0 cancels: Barbershop's dr0 = -0.43 puts a zero crossing inside the table."""
    scene = LOG_SCENES[name]
    cells = (np.arange(128, dtype=F32) + F32(0.5)) * F32(1.0 / 128.0)
    for lut, z in ((se.zlut(scene), cells), (se.zlut_dense(scene, 128), _dense_z(128))):
        ref, w = _world64(z, scene)
        err = np.abs(lut.astype(np.float64) - ref)
        assert (err <= se.ulp32(w)).all(), (err / se.ulp32(w)).max()
        print(f"{name}: max {float((err / se.ulp32(w)).max()):.3f} ulp of w, {float((err / se.ulp32(ref)).max()):.1f} ulp of the value")


@pytest.mark.parametrize("name", sorted(LOG_SCENES))
def test_depth_tables_against_the_oracle(name):
    """The oracle evaluates to_world in fp32 torch (pow included), so it is not the kernels' table: both are within 4 ulp of
    w of each other (absolute <= 4.8e-7 on Barbershop, 1.9e-6 on Pavillon).  Near Barbershop's zero crossing that is up to
    64 ulp of the value (fp32 cancellation in (w - 1) + dr0), so the bound is absolute, in units of w."""
    scene = LOG_SCENES[name]
    cells = (np.arange(128, dtype=F32) + F32(0.5)) * F32(1.0 / 128.0)
    oracle_dense = orc.stage2_sample(torch.zeros(1, 128), 0.0, 128, scene["depth_range"])["z"].numpy()[0]
    for lut, z, o in ((se.zlut(scene), cells, orc.log_to_world(torch.from_numpy(cells), scene["depth_range"]).numpy()),
                      (se.zlut_dense(scene, 128), _dense_z(128), oracle_dense)):
        _, w = _world64(z, scene)
        err = np.abs(lut.astype(np.float64) - o)
        assert (err <= 4 * se.ulp32(w)).all(), (err / se.ulp32(w)).max()
        assert err.max() <= 2e-6


def test_ndc_depth_tables_are_the_cell_centres():
    """FromClassifiedDepthAdaptiveNoDepthRange: the adaptive table is the cell centre itself, the dense one the lerp."""
    z = se.zlut(orc.SCENE_PAVILLON_NDC)
    np.testing.assert_array_equal(z, (np.arange(128, dtype=F32) + F32(0.5)) * F32(1.0 / 128.0))
    assert np.array_equal(z, orc.stage2_sample(torch.ones(1, 128), 0.5, 128, None, no_depth_range=True)["z"].numpy()[0])
    dense = orc.stage2_sample(torch.zeros(1, 128), 0.0, 128, None, no_depth_range=True)["z"].numpy()[0]
    np.testing.assert_array_equal(se.zlut_dense(orc.SCENE_PAVILLON_NDC, 128).view(np.uint32), dense.view(np.uint32))


def test_linspace_is_atens_rule():
    """linspace01 is ATen's per-element linspace rule (k * step below the half-way index, 1 - (K - k) * step from it).
    torch's vectorised CPU kernel continues a lane chunk that starts below the half-way index with k * step past it, so
    where 1 / K is inexact it can differ by 1 ulp; where 1 / K is a power of two every term is exact and the two agree bit
    for bit -- K = 128 among them, the only K dense mode takes."""
    for K in range(1, 257):
        ours = se.linspace01(K)
        ref = torch.linspace(0, 1, K + 1).numpy()
        diff = np.abs(ours.view(np.int32).astype(np.int64) - ref.view(np.int32))
        assert diff.max() <= 1, K
        if K & (K - 1) == 0:
            np.testing.assert_array_equal(ours.view(np.uint32), ref.view(np.uint32), err_msg=f"K={K}")
        assert ours[0] == 0 and ours[-1] == 1 and (np.diff(ours) > 0).all(), K
    K = 9                                       # the rule itself, written out once: ATen's symmetric evaluation
    step = F32(1) / F32(K)
    want = [F32(k) * step if k < 5 else F32(1) - F32(K - k) * step for k in range(K + 1)]
    np.testing.assert_array_equal(se.linspace01(K), np.array(want, F32))


def test_teeth_powf_depth_table():
    """A table built with powf on the fp32 base (instead of pow in double) differs from zlut in at least one cell of each
    shipped scene, so the GPU tests that compare z with zlut bit for bit catch it."""
    cells = (np.arange(128, dtype=F32) + F32(0.5)) * F32(1.0 / 128.0)
    for scene in LOG_SCENES.values():
        dr0, dr1 = F32(scene["depth_range"][0]), F32(scene["depth_range"][1])
        base = F32((float(dr1) - float(dr0)) + 1.0)
        bad = (np.power(base, cells, dtype=F32) - F32(1)) + dr0
        n = int((bad != se.zlut(scene)).sum())
        print(f"powf table: {n} of 128 cells differ")
        assert n >= 1


def test_stage2_packed_view_of_the_golden_cases():
    """stage2_packed on the oracle's selection is the golden cases' packed samples, and its z the golden z up to the
    to_world difference above."""
    for case in ("pav_k8_t0.2", "pav_k16_t0.15", "rand_k8_t0.2"):
        g = load_golden(case)
        m = g["meta"]
        scene = m["scene_params"]
        p = se.stage2_packed(orc.stage2_sample(torch.from_numpy(g["raw0"]), m["thr"], m["K"], scene["depth_range"]),
                             se.zlut(scene))
        mask = np.isfinite(g["z_nan"])
        np.testing.assert_array_equal(p["count"], mask.sum(1))
        np.testing.assert_array_equal(p["offset"], np.cumsum(mask.sum(1)) - mask.sum(1))
        np.testing.assert_array_equal(p["ray"], np.nonzero(mask)[0])
        np.testing.assert_allclose(p["z"], g["z_nan"][mask], rtol=0, atol=2e-6)
        assert p["total"] == mask.sum() and p["ray"].dtype == np.int32 and p["z"].dtype == F32


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


# ------------------------------------------------------------------------------------- stage-5 per-ray and padded outputs
@pytest.mark.parametrize("case", ["pav_k8_t0.2", "pav_k8_t0.5", "pav_k16_t0.15", "shaped_k8_t0.2", "rand_k8_t0.2",
                                  "ndc_k16_t0.15"])
def test_stage5_aux_emulation_matches_the_oracle(case):
    """alpha, z_vals, acc_map, disp_map and depth_est of both composites against the reference's tensors (golden alpha,
    z_vals, depth_est) and the oracle's composite (acc, disp) on the same inputs."""
    g = load_golden(case)
    m = g["meta"]
    K, scene = m["K"], m["scene_params"]
    mask, _, z = _packed(g, K)
    cnt = mask.sum(1)
    off = np.concatenate([[0], np.cumsum(cnt)[:-1]])
    o2 = orc.stage2_sample(torch.from_numpy(g["raw0"]), m["thr"], K, scene["depth_range"], no_depth_range=bool(scene.get("use_ndc")))
    zp = o2["zp"].numpy()[mask]
    raw1 = g["raw1_pad"].reshape(-1, 4)[mask.flatten()]
    comp = orc.stage5_composite(torch.from_numpy(raw1), torch.from_numpy(z), o2["zp"].float(), torch.from_numpy(mask.flatten()),
                                mask.shape[0], K)
    for fn in (se.stage5_thread, se.stage5_warp):
        out = fn(_sig32(raw1), zp, z, off, cnt, K)
        np.testing.assert_allclose(out["alpha"], g["alpha"], rtol=0, atol=1e-6)
        np.testing.assert_array_equal(out["z_vals"], g["z_nan"])          # NaN at the same places
        np.testing.assert_allclose(out["acc_map"], comp["acc"].numpy(), rtol=0, atol=2e-6)
        # disparity is ill-conditioned where depth_map / acc is tiny, so the rule is checked on the oracle's own inputs
        _assert_bits_equal(se.disp_map(comp["depth_map"].numpy(), comp["acc"].numpy()), comp["disp"].numpy())
        v, bound = se.depth_est_f64(out["depth_map"], scene)
        np.testing.assert_allclose(v, g["depth_est"][:, 0], rtol=0, atol=2e-6)
        ref = out["depth_map"] if scene.get("use_ndc") else orc.log_from_world(torch.from_numpy(out["depth_map"]), scene["depth_range"]).numpy()
        assert (np.abs(v - ref) <= bound + 4 * se.ulp32(ref)).all()


def test_stage5_dense_emulation_matches_the_oracle():
    """The dense variant against the oracle's dense composite (mapping None, zp = raw0, z = the dense table)."""
    rng = np.random.default_rng(12)
    n, scene = 200, orc.SCENE_BARBERSHOP
    raw0 = rng.uniform(-0.2, 1.2, (n, 128)).astype(F32)
    raw1 = rng.standard_normal((n * 128, 4)).astype(F32)
    lut = se.zlut_dense(scene, 128)
    out = se.stage5_dense(_sig32(raw1), raw0, lut)
    ref = orc.stage5_composite(torch.from_numpy(raw1), torch.from_numpy(np.tile(lut, n)), torch.from_numpy(raw0), None, n, 128)
    for k, rk in (("rgb", "rgb"), ("weights", "weights"), ("alpha", "alpha"), ("acc_map", "acc")):
        np.testing.assert_allclose(out[k], ref[rk].numpy(), rtol=0, atol=2e-6, err_msg=k)
    np.testing.assert_allclose(out["depth_map"], ref["depth_map"].numpy(), rtol=0, atol=2e-5)
    np.testing.assert_array_equal(out["z_vals"], np.tile(lut, (n, 1)))


def test_z_vals_of_a_live_sample_at_zero_is_nan_except_in_dense_mode():
    """features.py:546-547 sets every slot of the restored z == 0 to NaN, live samples at z = +-0 included; the dense path
    stores its z unchanged.  depth_map still uses z = 0 (adaptive_raw2outputs reads its own restored_z)."""
    sig = np.full((4, 4), 0.5, F32)
    zp = np.ones(4, F32)
    z = np.array([0.0, -0.0, 1.5, 0.0], F32)
    for fn in (se.stage5_thread, se.stage5_warp):
        out = fn(sig, zp, z, [0, 3], [3, 1], 4)
        assert np.isnan(out["z_vals"][0, [0, 1, 3]]).all() and out["z_vals"][0, 2] == F32(1.5)
        assert np.isnan(out["z_vals"][1]).all()
        assert out["z_vals"].view(np.uint32)[np.isnan(out["z_vals"])].tolist() == [0x7fc00000] * 7
    lut = np.zeros(128, F32)
    assert (se.stage5_dense(np.full((128, 4), 0.5, F32), np.ones((1, 128), F32), lut)["z_vals"] == 0).all()


def _torch_disp(dm, acc):
    dm, acc = torch.from_numpy(np.asarray(dm, F32)), torch.from_numpy(np.asarray(acc, F32))
    return (1.0 / torch.max(1e-10 * torch.ones_like(dm), dm / acc)).numpy()


def _assert_bits_equal(a, b):
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    np.testing.assert_array_equal(np.isnan(a), np.isnan(b))
    fin = ~np.isnan(a)
    np.testing.assert_array_equal(a[fin].view(np.uint32), b[fin].view(np.uint32))


def test_disp_map_is_torch_max():
    """disp_map equals 1 / torch.max(1e-10, dm / acc) bit for bit: 0 / 0, x / 0, +-inf quotients, negative acc, quotients
    around 1e-10, denormals, and NaN inputs.  The fmaxf form differs exactly where the quotient is NaN."""
    tiny, den = F32(1e-10), F32(2.0 ** -140)
    vals = np.array([0.0, -0.0, 1.0, -1.0, 0.5, 3.0, np.inf, -np.inf, np.nan, tiny, np.nextafter(tiny, F32(0)),
                     np.nextafter(tiny, F32(1)), den, -den, 1e30, 7.25], F32)
    dm, acc = (a.ravel() for a in np.meshgrid(vals, vals))
    rng = np.random.default_rng(5)
    dm = np.concatenate([dm, rng.standard_normal(5000).astype(F32) * 10])
    acc = np.concatenate([acc, rng.uniform(-0.5, 1.5, 5000).astype(F32)])
    ours, want = se.disp_map(dm, acc), _torch_disp(dm, acc)
    _assert_bits_equal(ours, want)
    assert np.isnan(se.disp_map(F32(0), F32(0)))
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        old = F32(1) / np.fmax(F32(1e-10), dm / acc)
    assert not np.array_equal(np.isnan(old), np.isnan(want))          # the fmaxf form gives 1e10 at 0 / 0


def _saturatef(x):
    """__saturatef (CUDA Math API): x clamped to [+0, 1], NaN -> +0."""
    return F32(0) if np.isnan(x) or x <= 0 else min(F32(x), F32(1))


def test_rgba8_is_the_viewers_compiled_clamp():
    """rgba8 on NaN, +-inf, +-0, every k / 255 and its fp32 neighbours, 1 - ulp, and values outside [0, 1], against a
    per-value trunc(__saturatef(x) * 255).  nvcc compiles helper_math.h's clamp fmaxf(0, fminf(x, 1)) -- and the other
    order too -- to one FADD.SAT, so the viewer's NaN pixel is 0, not the 255 the C semantics of the source would give."""
    ks = (np.arange(256, dtype=np.float64) / 255.0).astype(F32)
    x = np.concatenate([np.array([np.nan, -np.nan, np.inf, -np.inf, 0.0, -0.0, 1.0, np.nextafter(F32(1), F32(0)), 1.5, -0.25,
                                  2.0 ** -149, -2.0 ** -149, 1e30], F32),
                        ks, np.nextafter(ks, F32(2)), np.nextafter(ks, F32(-1))]).astype(F32)
    x = np.concatenate([x, np.zeros((-len(x)) % 3, F32)]).reshape(-1, 3)
    got = se.rgba8(x)
    want = np.array([[int(np.trunc(_saturatef(v) * F32(255))) for v in row] + [255] for row in x], np.uint8)
    np.testing.assert_array_equal(got, want)
    assert got[0, 0] == 0 and got[0, 1] == 0 and got[0, 2] == 255 and got[1, 0] == 0         # NaN, NaN, inf, -inf
    assert set(np.unique(se.rgba8(ks.reshape(-1, 1).repeat(3, 1))[:, 0])) == set(range(256))
