"""The SIMT stages against their fp32-faithful emulation (oracle/stage_emulation.py): stage 0, stage 3 and the stage-5
composites bit for bit, and every sine / cosine of the positional encoding bounded against float64.

What is exact and what is bounded:
  * positions, directions, the encodings' identity columns, ray_o / ray_d: every operation is an explicit
    round-to-nearest intrinsic or fma, so assert_array_equal against the emulation;
  * encoding anchor bands (f % 5 == 0, sincosf): within 2 ulp of float64 -- sincosf's documented maximum error (CUDA C++
    Programming Guide, single-precision mathematical functions);
  * encoding recurrence bands: bit-equal to the emulated double-angle recurrence seeded with the kernel's own anchors, and
    within the per-band bound se.recurrence_band_bounds() derives on the CPU from anchors perturbed by up to 2 ulp;
  * stage 5 with logits in {-200, 0, 200} (expf gives inf / 1 / 0 exactly, so every sigmoid is 0, 1/2 or 1): rgb,
    weights and depth bit for bit; with general logits within the operation-count bound _composite_f64 derives."""
import numpy as np
import pytest
import torch

from oracle import adanerf_oracle as orc
from oracle import stage_emulation as se

pytestmark = pytest.mark.gpu

F32, F64 = np.float32, np.float64
U = 2.0 ** -24
W = H = 800
SCENES = {"barbershop": orc.SCENE_BARBERSHOP, "pavillon": orc.SCENE_PAVILLON, "pavillon_ndc": orc.SCENE_PAVILLON_NDC}


def _renderer(scene, sd0=None):
    from adanerf_b200 import Renderer
    return Renderer(scene, device=0, sampling_net=sd0)


def _rot(kind):
    if kind == "identity":
        return np.eye(3, dtype=F32)
    yaw, pitch = np.radians(35.0), np.radians(-20.0)
    ry = np.array([[np.cos(yaw), -np.sin(yaw), 0], [np.sin(yaw), np.cos(yaw), 0], [0, 0, 1]])
    rp = np.array([[1, 0, 0], [0, np.cos(pitch), -np.sin(pitch)], [0, np.sin(pitch), np.cos(pitch)]])
    return (ry @ rp).astype(F32)


def _pose(scene, kind):
    """The view-cell centre, just inside the view-cell sphere, or outside it (where rays miss the sphere: delta < 0)."""
    c = np.asarray(scene["view_cell_center"], F64)
    r = np.linalg.norm(np.asarray(scene["view_cell_size"], F64) / 2)
    u = np.array([0.6, -0.7, 0.4]) / np.linalg.norm([0.6, -0.7, 0.4])
    return (c + {"centre": 0.0, "surface": 0.98 * r, "outside": 1.7 * r}[kind] * u).astype(F32)


def _grazing_dirs(scene, pose, rot, n=4096):
    """Directions (camera frame) whose rotated ray touches the view-cell sphere within a relative 1e-5 of the tangent."""
    c = np.asarray(scene["view_cell_center"], F64)
    r = np.linalg.norm(np.asarray(scene["view_cell_size"], F64) / 2)
    a = c - pose.astype(F64)
    D = np.linalg.norm(a)
    a /= D
    b1 = np.cross(a, [0.0, 0.0, 1.0])
    b1 /= np.linalg.norm(b1)
    b2 = np.cross(a, b1)
    rng = np.random.default_rng(7)
    th = np.arcsin(r / D) * (1 + rng.uniform(-1e-5, 1e-5, n))
    ph = rng.uniform(0, 2 * np.pi, n)
    g = np.cos(th)[:, None] * a + np.sin(th)[:, None] * (np.cos(ph)[:, None] * b1 + np.sin(ph)[:, None] * b2)
    return (g @ rot.astype(F64)).astype(F32)          # R^T g: the kernel rotates it back


def check_encoding(block, v, L, what):
    """block: the kernel's [M, 3 + 6L] encoding of v [M, 3] (the emulated input, itself compared bit for bit)."""
    np.testing.assert_array_equal(block[:, :3], v, err_msg=f"{what}: identity columns")
    np.testing.assert_array_equal(block, se.posenc3(v, L, anchors=block), err_msg=f"{what}: recurrence bands")
    fin = np.isfinite(v).all(1)
    got = block[fin, 3:].astype(F64).reshape(-1, L, 2, 3)
    ref = se.posenc_f64(v[fin], L)[:, 3:].reshape(-1, L, 2, 3)
    err = np.abs(got - ref)
    for f in range(0, L, se.ANCHOR_EVERY):
        ulps = err[:, f] / se.ulp32(ref[:, f])
        assert ulps.max(initial=0) <= 2.0, f"{what}: sincosf band {f} off by {ulps.max():.2f} ulp"
    band = err.max(axis=(0, 2, 3), initial=0)
    bound = se.recurrence_band_bounds()[:L]
    assert (band <= bound).all(), f"{what}: band errors {band} exceed {bound}"


# ------------------------------------------------------------------------------------------------------ stage 0
@pytest.mark.parametrize("pose_kind,rot_kind", [("centre", "identity"), ("centre", "yaw_pitch"), ("surface", "yaw_pitch"),
                                                ("outside", "yaw_pitch")])
@pytest.mark.parametrize("scene_name", list(SCENES))
def test_stage0_bit_exact(scene_name, pose_kind, rot_kind):
    """A whole 800x800 frame (plus, from outside the sphere, rays grazing it) through generate_ray_directions and stage 0:
    the directions, ray_o, ray_d and the identity columns of both encoded blocks equal the emulation bit for bit."""
    scene = SCENES[scene_name]
    r = _renderer(scene)
    pose, rot = _pose(scene, pose_kind), _rot(rot_kind)
    dirs = r.generate_ray_directions(W, H).cpu().numpy()
    np.testing.assert_array_equal(dirs, se.pixel_dir(W, H, scene["fov"]))
    if pose_kind == "outside":
        dirs = np.concatenate([dirs, _grazing_dirs(scene, pose, rot)])
    x0, ro, rd = (t.cpu().numpy() for t in r.stage0(pose, rot, torch.from_numpy(dirs)))
    e_ro, e_rd, e_x0 = se.stage0(pose, rot, dirs, scene)
    np.testing.assert_array_equal(rd, e_rd)
    np.testing.assert_array_equal(ro, e_ro)
    k = se.scene_constants(scene)
    nd = 3 + 6 * k["nfd0"]
    assert x0.shape[1] == nd + 3 + 6 * k["nfp0"]
    check_encoding(x0[:, :nd], e_x0[:, :3], k["nfd0"], "direction block")
    check_encoding(x0[:, nd:], e_ro, k["nfp0"], "position block")
    udot, delta = se.sphere_delta(pose, e_rd, scene)
    if pose_kind == "outside":   # the clamp is exercised, and so are rays within a hair of the tangent
        assert (delta < 0).sum() > 1000 and (np.abs(delta[-4096:]) < 1e-3 * udot[-4096:] ** 2).sum() > 100
    r.close()


# ------------------------------------------------------------------------------------------------------ stage 3
def _check_stage3(r, scene, ro, rd, ray, z, what):
    x1 = r.stage3(torch.from_numpy(ro), torch.from_numpy(rd), torch.from_numpy(ray.astype(np.int32)),
                  torch.from_numpy(z)).cpu().numpy()
    pos, d = se.sample_inputs(scene, ro, rd, ray, z)
    np.testing.assert_array_equal(x1[:, :3], pos, err_msg=f"{what}: positions")
    np.testing.assert_array_equal(x1[:, 63:66], d, err_msg=f"{what}: directions")
    check_encoding(x1[:, :63], pos, 10, f"{what}: position block")
    check_encoding(x1[:, 63:], d, 4, f"{what}: direction block")
    return pos


def test_stage3_full_frame_bit_exact():
    """A full 800x800 frame's packed samples (thr 0.2, K 8: ~5 M samples, shaped sampling net) through stage 3, compared
    in chunks of 2^19 samples."""
    scene = orc.SCENE_BARBERSHOP
    sd0, _ = orc.make_weights("shaped", seed=0)
    r = _renderer(scene, sd0)
    pose, rot = _pose(scene, "surface"), _rot("yaw_pitch")
    x0, ro_d, rd_d = r.stage0(pose, rot, r.generate_ray_directions(W, H))
    s2 = r.stage2(r.mlp0(x0), 0.2, 8)
    M = s2["total"]
    assert M > 3_000_000, M
    ro, rd = ro_d.cpu().numpy(), rd_d.cpu().numpy()
    ray, z = s2["ray"].cpu().numpy(), s2["z"].cpu().numpy()
    step = 1 << 19
    for a in range(0, M, step):
        _check_stage3(r, scene, ro, rd, ray[a:a + step], z[a:a + step], f"samples {a}..")
    r.close()


@pytest.mark.parametrize("scene_name", ["barbershop", "pavillon_ndc"])
def test_stage3_edges_bit_exact(scene_name):
    """Samples at the view-cell centre (0/0 -> NaN, like the reference), z = 0, large and negative z (with NDC, 2^9 x past
    sincosf's slow-path threshold |x| > 105615), and 1, 127, 129 samples around the 128-sample tile."""
    scene = SCENES[scene_name]
    r = _renderer(scene)
    rng = np.random.default_rng(21)
    dirs = se.pixel_dir(W, H, scene["fov"])[rng.integers(0, W * H, 300)]
    _, rd, _ = se.stage0(_pose(scene, "surface"), _rot("yaw_pitch"), dirs, scene)
    c = np.asarray(scene["view_cell_center"], F32)
    ro = (c + rng.uniform(-0.3, 0.3, (300, 3))).astype(F32)
    ro[0] = c                                                   # ray 0 starts at the centre
    n = 3000
    ray = rng.integers(0, 300, n)
    z = rng.uniform(0.01, 8.0, n).astype(F32)
    z[:600] = rng.choice(np.array([0.0, -0.0, 300.0, 1000.0, -500.0, 4096.5], F32), 600)
    ray[:4], z[:4] = 0, 0.0                                     # centre samples
    z[4:20] = 0.0
    pos = _check_stage3(r, scene, ro, rd, ray, z, "edges")
    if scene.get("use_ndc"):
        assert (np.abs(pos) * 512 > 105615).any()
    else:
        assert np.isnan(pos[:4]).all()
    for m in (1, 127, 128, 129):
        _check_stage3(r, scene, ro, rd, ray[-m:], z[-m:], f"{m} samples")
    r.close()


# ------------------------------------------------------------------------------------------------------ stage 5
@pytest.fixture(scope="module")
def bare():
    r = _renderer(orc.SCENE_BARBERSHOP)
    yield r
    r.close()


def _layout(K, rng, n_random=200):
    """Per-ray counts 0, 1, K and the 32-sample block edges, then random ones; packed offsets."""
    edges = sorted({c for c in (0, 1, 2, 31, 32, 33, 63, 64, 65, 95, 96, 97, 127, 128, K - 1, K) if 0 <= c <= K})
    cnt = np.concatenate([np.repeat(edges, 4), rng.integers(0, K + 1, n_random)]).astype(np.int32)
    return (np.cumsum(cnt) - cnt).astype(np.int32), cnt


def _sig64(x):
    return 1.0 / (1.0 + np.exp(-np.asarray(x, F64)))


@pytest.mark.parametrize("K", [1, 2, 8, 9, 16, 17, 31, 32, 33, 63, 64, 65, 100, 127, 128])
def test_stage5_bit_exact_with_exact_sigmoids(bare, K):
    """K <= 32: stage5_thread_kernel, K > 32: stage5_warp_kernel.  zp and z are arbitrary fp32 values (zp > 1, < 0, = 0,
    z of any sign and size), so the transmittance leaves [0, 1] and may overflow: the bits still have to agree."""
    rng = np.random.default_rng(K)
    off, cnt = _layout(K, rng)
    M = int(cnt.sum())
    logits = rng.choice(np.array([-200.0, 0.0, 200.0], F32), (M, 4))
    zp = np.where(rng.random(M) < 0.4, rng.choice(np.array([0.0, 1.0, 2.0, -0.75, 0.5, 1.5, -0.0], F32), M),
                  (rng.standard_normal(M) * 1.5).astype(F32)).astype(F32)
    z = (rng.standard_normal(M) * 10.0 ** rng.integers(-3, 4, M)).astype(F32)
    sig = _sig64(logits).astype(F32)
    assert set(np.unique(sig).tolist()) == {0.0, 0.5, 1.0}
    out = bare.stage5(torch.from_numpy(logits), torch.from_numpy(zp), torch.from_numpy(z), torch.from_numpy(off),
                      torch.from_numpy(cnt), K)
    emu = se.stage5(sig, zp, z, off, cnt, K)
    for k in ("rgb", "weights", "depth_map"):
        np.testing.assert_array_equal(out[k].cpu().numpy(), emu[k], err_msg=k)


def _composite_f64(logits, zp, z, off, cnt, K):
    """The composite in float64 with a first-order bound on the fp32 kernels' error, u = 2^-24, all quantities >= 0:
      sigmoid: expf within 2 ulp (<= 4u relative; CUDA C++ Programming Guide), 1 + e and 1 / (.) one rounding each -> 6u s;
      alpha = s_a zp: e_a = zp e_s + u alpha;  f = (1 - alpha) + 1e-10: e_f = e_a + u |1 - alpha| + u f;
      T_j = prod_{i<j} f_i by any product tree: every rounding of a partial product costs at most u T_j once the other
      factors (<= 1) multiply it, and T_j's tree has at most j + 1 multiplies -> e_T = sum_{i<j} e_f(i) T_i + (j + 1) u T_j;
      w = alpha T: e_w = e_a T + alpha e_T + u w;  term = w s: e_w s + w e_s + u term;
      sum of n terms in any order of depth <= n + 9 (thread: n sequential adds; warp: <= 4 per lane + 5 butterfly levels):
      (n + 9) u sum(term); acc_map = sum w the same way.  Returns (rgb, weights, alpha, depth_map, acc_map) and their
      bounds."""
    n = cnt.shape[0]
    eps = float(se.EPS_T)
    T, S = np.ones(n), np.zeros(n)
    rgb, e_rgb = np.zeros((n, 3)), np.zeros((n, 3))
    dm, e_dm, sum_rgb, sum_dm = np.zeros(n), np.zeros(n), np.zeros((n, 3)), np.zeros(n)
    w_out, e_w_out = np.zeros((n, K)), np.zeros((n, K))
    a_out, e_a_out = np.zeros((n, K)), np.zeros((n, K))
    acc, e_acc = np.zeros(n), np.zeros(n)
    for j in range(K):
        live = j < cnt
        idx = np.where(live, off + j, 0)
        s = _sig64(logits[idx])
        e_s = 6 * U * s
        a = s[:, 3] * zp[idx]
        e_a = zp[idx] * e_s[:, 3] + U * a
        f = (1.0 - a) + eps
        e_f = e_a + U * np.abs(1.0 - a) + U * f
        e_T = S + (j + 1) * U * T
        w = a * T
        e_w = e_a * T + a * e_T + U * w
        term, zt = w[:, None] * s[:, :3], w * z[idx]
        upd = lambda acc, x: np.where(live[:, None] if acc.ndim == 2 else live, acc + x, acc)
        rgb, sum_rgb = upd(rgb, term), upd(sum_rgb, term)
        e_rgb = upd(e_rgb, e_w[:, None] * s[:, :3] + w[:, None] * e_s[:, :3] + U * term)
        dm, sum_dm = upd(dm, zt), upd(sum_dm, zt)
        e_dm = upd(e_dm, e_w * z[idx] + U * zt)
        acc, e_acc = upd(acc, w), upd(e_acc, e_w)
        w_out[:, j], e_w_out[:, j] = np.where(live, w, 0), np.where(live, e_w, 0)
        a_out[:, j], e_a_out[:, j] = np.where(live, a, 0), np.where(live, e_a, 0)
        S = np.where(live, S + e_f * T, S)
        T = np.where(live, T * f, T)
    depth = (cnt + 9) * U
    return (dict(rgb=rgb, weights=w_out, alpha=a_out, depth_map=dm, acc_map=acc),
            dict(rgb=1.01 * (e_rgb + depth[:, None] * sum_rgb), weights=1.01 * e_w_out, alpha=1.01 * e_a_out,
                 depth_map=1.01 * (e_dm + depth * sum_dm), acc_map=1.01 * (e_acc + depth * acc)))


@pytest.mark.parametrize("K", [8, 17, 32, 33, 64, 128])
def test_stage5_general_logits_within_operation_count_bound(bare, K):
    rng = np.random.default_rng(100 + K)
    off, cnt = _layout(K, rng, n_random=2000)
    M = int(cnt.sum())
    logits = np.clip(rng.standard_normal((M, 4)) * 4, -16, 16).astype(F32)
    zp, z = rng.uniform(0, 1, M).astype(F32), rng.uniform(0, 10, M).astype(F32)
    out = bare.stage5(torch.from_numpy(logits), torch.from_numpy(zp), torch.from_numpy(z), torch.from_numpy(off),
                      torch.from_numpy(cnt), K)
    ref, bound = _composite_f64(logits, zp.astype(F64), z.astype(F64), off, cnt, K)
    for k in ("rgb", "weights", "depth_map"):
        err = np.abs(out[k].cpu().numpy().astype(F64) - ref[k])
        worst = (err / np.maximum(bound[k], 1e-300)).max()
        print(f"K={K} {k}: max err {err.max():.3e}, max err / bound {worst:.3f}")
        assert (err <= bound[k]).all(), k
