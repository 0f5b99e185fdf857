"""oracle/stage_emulation.py on the CPU: fma32 is a correctly rounded fp32 fma, the emulation restates the reference (the
oracle and the golden cases, at the tolerances the reference comparisons use), and deliberately wrong variants of it fail
the checks tests/test_stage_kernels_exact.py applies to the kernels (teeth)."""
from fractions import Fraction

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import adanerf_oracle as orc
from oracle import donerf_oracle as dno
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


def test_linspace_is_torch_linspace():
    """linspace01 is torch.linspace(0, 1, K + 1) on the CPU bit for bit at every length 2 ... 259 (the sampler's u takes
    lengths K + 2 <= 130, its cell edges and the dense table 129): k * step below the half-way index, fma(-step, K - k, 1)
    from it.  The two-rounding form 1 - (K - k) * step differs at most lengths, though not at 129."""
    n_two = 0
    for K in range(1, 259):
        ours = se.linspace01(K)
        ref = torch.linspace(0, 1, K + 1).numpy()
        np.testing.assert_array_equal(ours.view(np.uint32), ref.view(np.uint32), err_msg=f"length {K + 1}")
        assert ours[0] == 0 and ours[-1] == 1 and (np.diff(ours) > 0).all(), K
        step, k = F32(1) / F32(K), np.arange(K + 1)
        two = np.where(k < (K + 1) // 2, k.astype(F32) * step, F32(1) - (K - k).astype(F32) * step).astype(F32)
        n_two += not np.array_equal(two, ref)
        if K == 128:
            np.testing.assert_array_equal(two, ref)
    assert n_two > 200, n_two
    K = 9                                       # the rule itself, written out once
    step = F32(1) / F32(K)
    want = [F32(k) * step if k < 5 else se.fma32(-step, F32(K - k), F32(1)) for k in range(K + 1)]
    np.testing.assert_array_equal(se.linspace01(K), np.array(want, F32))
    assert any(not np.array_equal(se.linspace01(k, symmetric=False), se.linspace01(k)) for k in range(2, 130))


@pytest.mark.parametrize("name", sorted(LOG_SCENES))
def test_dense_table_keeps_its_bits(name):
    """zlut_dense(scene, 128) is the table of the two-rounding linspace: 1 / 128 is a power of two, so both forms are exact."""
    scene = LOG_SCENES[name]
    t = (np.arange(128, dtype=F32) * F32(1.0 / 128)).astype(F32) + F32(0.5 / 128)
    z = F32(0.001) * (F32(1) - t) + F32(1.0) * t
    np.testing.assert_array_equal(se.zlut_dense(scene, 128).view(np.uint32), se._to_world(z, scene).view(np.uint32))


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


# ------------------------------------------------------------------------------------------------- fixed-K sampler
DONERF_CASES = [("rand", t, K) for t in ("sigmoid", "softmax") for K in (1, 4, 8, 16)] + \
               [("pav", t, K) for t in ("sigmoid", "softmax") for K in (4, 16)]
TRANSFORM = {"sigmoid": 1, "softmax": 2}


def _expf64(x):
    """Correctly rounded expf through float64."""
    with np.errstate(over="ignore"):
        return np.exp(np.asarray(x, F32).astype(np.float64)).astype(F32)


def _pow64(base, x):
    return np.power(base, np.asarray(x, F32).astype(np.float64))


def _powf(base, x):
    return np.power(F32(base), np.asarray(x, F32), dtype=F32)


def _donerf_fixture(nets, tname, K):
    from adanerf_b200.synthetic import load_npz
    import os
    g = load_npz(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", f"donerf_{nets}_{tname}_k{K}.npz"))
    return g, orc.SCENE_PAVILLON if nets == "pav" else orc.SCENE_BARBERSHOP


def _pdf_edge_rows():
    """raw0 rows [R,128] at the sampler's edges: constant rows (exact ties), one-hot rows (+-200), two spikes with long
    clamped runs between them (cells 0 and 127 among them), all -200, softmax rows with x - m in [-104, -87] (subnormal
    exp) and below -104 (exp = 0), +-1e30 and -0.0, rows holding +-inf or NaN, and plain random rows."""
    R = [np.full(128, v) for v in (0.0, 3.5, -200.0, 200.0, 1e30, -1e30, -0.0)]
    for c in (0, 1, 63, 64, 127):
        for hi, lo in ((200.0, -200.0), (-200.0, 200.0)):
            r = np.full(128, lo)
            r[c] = hi
            R.append(r)
    for a, b in ((0, 127), (0, 64), (5, 90), (126, 127), (0, 1), (31, 96)):
        r = np.full(128, -200.0)
        r[[a, b]] = 200.0
        R.append(r)
        r = np.full(128, -200.0)
        r[a], r[b] = 200.0, 0.0
        R.append(r)
    rng = np.random.default_rng(11)
    for lo, hi in ((-104.0, -87.0), (-150.0, -104.0), (-110.0, -80.0)):
        r = rng.uniform(lo, hi, 128)
        r[rng.integers(128)] = 0.0
        R.append(r)
    R.extend(rng.choice([1e30, -1e30, -0.0, 0.0], (4, 128)))
    for v in (np.inf, -np.inf, np.nan):
        for c in (0, 77, 127):
            r = rng.standard_normal(128) * 3
            r[c] = v
            R.append(r)
        R.append(np.full(128, v))
    r = rng.standard_normal(128)
    r[3], r[90] = np.inf, -np.inf
    R.append(r)
    r = np.full(128, -200.0)
    r[[10, 20]] = np.inf
    R.append(r)
    for s in (0.01, 1, 10, 50):
        R.extend(rng.standard_normal((8, 128)) * s)
    with np.errstate(over="ignore"):
        return np.asarray(R, F32)


@pytest.mark.parametrize("case", DONERF_CASES, ids=[f"{n}-{t}-k{k}" for n, t, k in DONERF_CASES])
def test_pdf_sample_emulation_matches_the_oracle(case):
    """With correctly rounded transcendentals the emulation is the reference's z (the fixtures, which
    donerf_oracle.pdf_sample reproduces bit for bit) up to the documented deviations: within 10 ulp of the power w on the
    Pavillon net's peaked distributions; on the random nets' flat ones, where t = (u - c0) / denom amplifies a last-bit
    cdf difference, within 256 ulp of w and 1e-5 of the warped range.  z ascends per ray."""
    g, scene = _donerf_fixture(*case)
    K = case[2]
    z = se.pdf_sample(g["raw0"], K, TRANSFORM[case[1]], scene, _expf64, _pow64)
    assert z.shape == g["z"].shape and (np.diff(z, axis=1) >= 0).all()
    dr0, dr1 = (float(F32(v)) for v in scene["depth_range"])
    w = g["z"].astype(np.float64) - dr0 + 1.0
    ulps = np.abs(z.astype(np.float64) - g["z"]) / se.ulp32(w)
    du = np.abs(np.log(z.astype(np.float64) - dr0 + 1.0) - np.log(w)) / np.log(dr1 - dr0 + 1.0)
    print(f"{case}: {100 * (ulps > 0).mean():.1f} % of z differ, at most {ulps.max():.0f} ulp of w, {du.max():.2g} of the warped range")
    assert ulps.max() <= (10 if case[0] == "pav" else 256) and du.max() <= 1e-5


def test_pdf_search_shortcut_is_the_binary_search():
    """_search's counting shortcut (non-decreasing, NaN-free rows) equals the kernel's binary search and np.searchsorted
    per row, for right=True and False; rows with NaN or a decreasing step take the search itself."""
    rng = np.random.default_rng(3)
    raw = np.concatenate([_pdf_edge_rows(), (rng.standard_normal((400, 128)) * rng.choice([0.1, 1, 5, 30], (400, 1)))])
    for tr in (1, 2):
        cdf = se.pdf_cdf(se.pdf_transform(raw.astype(F32), tr, _expf64))
        mono = ~np.isnan(cdf).any(1) & (np.diff(cdf, axis=1) >= 0).all(1)
        assert (~mono).sum() >= 4 and mono.sum() > 400
        for K in (1, 7, 33, 128):
            u = se.linspace01(K + 1)[1:K + 1]
            for right in (True, False):
                got, lit = se._search(cdf, u, right), se.binary_search(cdf, u, right)
                np.testing.assert_array_equal(got, lit)
                ref = np.stack([np.searchsorted(c, u, side="right" if right else "left") for c in cdf[mono]])
                np.testing.assert_array_equal(got[mono], ref)


def test_pdf_edge_rows_keep_nan_in_their_ray():
    """Rows holding +-inf or NaN: the emulation's NaN samples are the oracle's, sample for sample, and no finite row has one."""
    raw = _pdf_edge_rows()
    finite = np.isfinite(raw).all(1)
    for tr in (1, 2):
        for K in (1, 7, 33, 128):
            z = se.pdf_sample(raw, K, tr, orc.SCENE_PAVILLON, _expf64, _pow64)
            ref = dno.pdf_sample(torch.from_numpy(raw), K, tr, orc.SCENE_PAVILLON["depth_range"]).numpy()
            np.testing.assert_array_equal(np.isnan(z), np.isnan(ref))
            assert not np.isnan(z[finite]).any() and np.isnan(z).any()


SAMPLER_TEETH = {"fp32 cdf": dict(scan="fp32"), "fp32 sequential wsum": dict(wsum="fp32"), "right=False": dict(right=False),
                 "no clamp": dict(clamp=False), "j step linspace": dict(symmetric=False), "fp32 pow": dict(pow64=_powf)}


def test_teeth_sampler():
    """Each mutation of the sampler's emulation moves at least one z of the edge rows and the fixtures' raw0."""
    raw = np.concatenate([_pdf_edge_rows()] + [_donerf_fixture(*c)[0]["raw0"] for c in (("pav", "sigmoid", 16), ("rand", "softmax", 16))])
    moved = {k: 0 for k in SAMPLER_TEETH}
    for tr in (1, 2):
        for K in (7, 33, 128):
            good = se.pdf_sample(raw, K, tr, orc.SCENE_PAVILLON, _expf64, _pow64)
            for name, kw in SAMPLER_TEETH.items():
                kw = dict(dict(expf=_expf64, pow64=_pow64), **kw)
                bad = se.pdf_sample(raw, K, tr, orc.SCENE_PAVILLON, **kw)
                moved[name] += int((~((bad.view(np.int32) == good.view(np.int32)) | (np.isnan(bad) & np.isnan(good)))).sum())
    print("samples moved:", moved)
    assert all(v > 0 for v in moved.values()), moved


def test_teeth_density_composite():
    """tree=False and butterfly=False change the warp composite's outputs on the density path."""
    rng = np.random.default_rng(8)
    n, K = 300, 100
    raw1 = (rng.standard_normal((n * K, 4)) * 2).astype(F32)
    z = np.sort(rng.uniform(0.2, 8, (n, K)), axis=1).astype(F32).reshape(-1)
    rd = rng.standard_normal((n, 3)).astype(F32)
    alpha = se.density_alpha(raw1[:, 3], z, rd, K, _expf64)
    sig = _sig32(raw1[:, :3])
    args = (sig, None, z, np.arange(n) * K, np.full(n, K), K)
    good = se.stage5_warp(*args, alpha=alpha)
    for kw in (dict(tree=False), dict(butterfly=False)):
        bad = se.stage5_warp(*args, alpha=alpha, **kw)
        assert not np.array_equal(good["rgb"], bad["rgb"]), kw


@pytest.mark.parametrize("case", DONERF_CASES, ids=[f"{n}-{t}-k{k}" for n, t, k in DONERF_CASES])
def test_density_composite_emulation_matches_the_reference(case):
    """density_alpha + stage5_density on the fixtures' raw1 / z / rays_d against the reference's tensors (at
    test_donerf_gpu's tolerances: ATen's vectorised exp is not expf), z_vals = z, and K = 1 composites to nothing.  The
    thread and warp chains agree with each other to the same tolerance."""
    g, _ = _donerf_fixture(*case)
    K = case[2]
    n = g["ray_d"].shape[0]
    raw1, z = g["raw1"].reshape(n * K, 4), g["z"].reshape(-1)
    alpha = se.density_alpha(raw1[:, 3], z, g["ray_d"], K, _expf64)
    for fn in (se.stage5_thread, se.stage5_warp):
        out = fn(_sig32(raw1[:, :3]), None, z, np.arange(n) * K, np.full(n, K), K, alpha=alpha)
        np.testing.assert_array_equal(out["z_vals"], g["z"])
        if K == 1:
            assert (out["alpha"] == 0).all() and (out["rgb"] == 0).all() and (out["acc_map"] == 0).all()
            continue
        np.testing.assert_allclose(out["alpha"], g["alpha"], rtol=1e-5, atol=2e-6)
        np.testing.assert_allclose(out["weights"], g["weights"], rtol=1e-5, atol=2e-6)
        np.testing.assert_allclose(out["rgb"], g["rgb"], rtol=1e-5, atol=2e-6)
    assert se.stage5_density(_sig32(raw1[:, :3]), alpha, z, K)["z_vals"].shape == (n, K)


def test_density_alpha_rules():
    """relu keeps NaN, the last sample's distance is 1e10 |d|, repeated z with an inf density is 0 * inf = NaN, decreasing z
    gives alpha < 0, |d| = 0 gives alpha 0, K = 1 gives alpha 0."""
    a = np.array([np.nan, -1.0, 2.0, np.inf, 1.0, 1.0], F32)
    z = np.array([0.0, 1.0, 2.0, 4.0, 4.0, 3.5], F32)
    al = se.density_alpha(a, z, np.array([[0.0, 3.0, 4.0]], F32), 6, _expf64)
    assert np.isnan(al[0]) and al[1] == 0 and al[2] == F32(1) - _expf64(F32(-20.0)) and np.isnan(al[3])
    assert al[4] < 0 and al[5] == 1
    assert (se.density_alpha(a, z, np.zeros((1, 3), F32), 6, _expf64)[1:3] == 0).all()
    assert (se.density_alpha(a, z, np.ones((6, 3), F32), 1, _expf64) == 0).all()


def test_fixture_z_attribution():
    """Which documented deviation moves which fixture z bits.  Starting from torch's CPU sigmoid / softmax values, the
    kernel's placement is switched to the reference's one deviation at a time: torch.sum for the double warp sum, one
    sequential double cumsum for the warp scan, torch's fp32 pow for the double pow -- evaluated, as the reference does,
    on the [:, 1:-1] slice of the K + 2 samples (ATen's fp32 pow gives other bits on a contiguous tensor).  With the sum
    and the pow both switched every fixture bit is the reference's; the scan association moves none."""
    tsum = lambda w: torch.sum(torch.from_numpy(w), -1).numpy()
    counts, total = {}, 0

    def pow_ref(scene):
        dr = scene["depth_range"]

        def f(base, x):
            t = torch.zeros(x.shape[0], x.shape[1] + 2)
            t[:, 1:-1] = torch.from_numpy(np.asarray(x, F32))
            return ((dr[1] - dr[0] + 1) ** t[:, 1:-1]).numpy()
        return f

    for case in DONERF_CASES:
        g, scene = _donerf_fixture(*case)
        K = case[2]
        x = torch.from_numpy(g["raw0"])
        w = (torch.sigmoid(x) if case[1] == "sigmoid" else torch.softmax(x, -1)).numpy()
        total += g["z"].size
        for s in ("double", "torch.sum"):
            for c in ("warp", "seq"):
                cdf = se.pdf_cdf(w, wsum=tsum if s == "torch.sum" else "warp", scan=c)
                for p in ("double", "fp32"):
                    z = se.pdf_place(cdf, K, scene, pow_ref(scene) if p == "fp32" else _pow64)
                    key = (s, c, p)
                    counts[key] = counts.get(key, 0) + int((z.view(np.int32) != g["z"].view(np.int32)).sum())
    for k, v in counts.items():
        print(f"sum {k[0]:9s} scan {k[1]:4s} pow {k[2]:6s}: {v:5d} of {total} fixture z differ ({100 * v / total:.1f} %)")
    assert counts[("torch.sum", "warp", "fp32")] == 0 and counts[("torch.sum", "seq", "fp32")] == 0
    for s in ("double", "torch.sum"):
        for p in ("double", "fp32"):
            assert counts[(s, "warp", p)] == counts[(s, "seq", p)]
    assert counts[("double", "warp", "fp32")] > 0 and counts[("torch.sum", "warp", "double")] > 0
