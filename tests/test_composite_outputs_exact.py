"""Every output stage 5 writes, bit for bit: rgb, weights, alpha, z_vals, depth_map, acc_map, disp_map and the RGBA8 pixels
against the fp32-faithful emulation (oracle/stage_emulation.py), depth_est within logf's documented bound, in both
composite kernels and dense mode; then the same outputs of every render entry point against the stage entry points
composed by hand.

Buffers are pre-filled with a sentinel (bit pattern 0x7f7f7f7f, bytes 0x7f) so a slot a kernel or a chunk never writes
shows up.  NaN compares by position: the kernels' NaN payloads are the GPU's, the emulation's numpy's."""
import math

import numpy as np
import pytest
import torch

from oracle import adanerf_oracle as orc
from oracle import stage_emulation as se
from test_stage_kernels_exact import _composite_f64, _layout, _sig64

pytestmark = pytest.mark.gpu

F32, F64 = np.float32, np.float64
SENTINEL = 0x7f7f7f7f
AUX = ("weights", "alpha", "z_vals", "depth_map", "acc_map", "disp_map", "depth_est")
SCENES = {"log": orc.SCENE_BARBERSHOP, "ndc": orc.SCENE_PAVILLON_NDC}


def _renderer(scene, sd0=None, sd1=None):
    from adanerf_b200 import Renderer
    return Renderer(scene, device=0, sampling_net=sd0, shading_net=sd1)


def _filled(shape, dtype=torch.float32):
    t = torch.empty(shape, dtype=dtype, device="cuda")
    if dtype == torch.uint8:
        return t.fill_(0x7f)
    t.view(torch.int32).fill_(SENTINEL)
    return t


def _prefilled(n, K):
    out = {k: _filled((n, K) if k in ("weights", "alpha", "z_vals") else (n,)) for k in AUX}
    out.update(rgb=_filled((n, 3)), rgba8=_filled((n, 4), torch.uint8))
    return out


def _stage5(r, raw1, zp, z, off, cnt, K, dense=False):
    n = zp.shape[0] if dense else cnt.shape[0]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)) if a is not None else None
    return r.stage5(t(raw1), t(zp), t(z), t(off), t(cnt), K, aux=True, dense=dense, rgba8=True, out=_prefilled(n, K))


def _same(got, want, what):
    """Bit-equal, NaN at the same places (any payload)."""
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, what
    if got.dtype == np.uint8:
        np.testing.assert_array_equal(got, want, err_msg=what)
        return
    gn, wn = np.isnan(got), np.isnan(want)
    np.testing.assert_array_equal(gn, wn, err_msg=f"{what}: NaN positions")
    np.testing.assert_array_equal(got[~gn].view(np.uint32), want[~wn].astype(F32).view(np.uint32), err_msg=what)


def _check_epilogue(out, scene, what):
    """disp_map, rgba8 bit for bit and depth_est within its bound, as functions of the kernel's own depth_map / acc_map /
    rgb; every ray that takes the d <= 0 branch holds one and the same depth_est."""
    dm, acc, rgb = out["depth_map"], out["acc_map"], out["rgb"]
    _same(out["disp_map"], se.disp_map(dm, acc), f"{what}: disp_map")
    _same(out["rgba8"], se.rgba8(rgb), f"{what}: rgba8")
    de = out["depth_est"]
    if scene.get("use_ndc"):
        _same(de, dm, f"{what}: depth_est (NDC: the depth map)")
        return
    v, bound = se.depth_est_f64(dm, scene)
    fin = np.isfinite(v)
    err = np.abs(de[fin].astype(F64) - v[fin])
    assert (err <= bound[fin]).all(), f"{what}: depth_est off by {(err / bound[fin]).max():.2f} x its bound"
    _same(de[~fin], v[~fin].astype(F32), f"{what}: depth_est (inf / NaN)")
    with np.errstate(invalid="ignore"):
        clamped = (dm - F32(scene["depth_range"][0])) <= 0
    if clamped.any():
        assert np.unique(de[clamped].view(np.uint32)).size == 1, f"{what}: the d <= 0 branch is not one value"
        assert abs(float(de[clamped][0]) - math.log(float(F32(0.001) + F32(1))) / float(se.log_range(scene))) <= bound[clamped][0]
    return clamped.sum()


def _check_all(out, emu, scene, what):
    out = {k: v.cpu().numpy() for k, v in out.items()}
    for k in ("rgb", "weights", "alpha", "z_vals", "depth_map", "acc_map"):
        _same(out[k], emu[k], f"{what}: {k}")
    return _check_epilogue(out, scene, what)


# ------------------------------------------------------------------------------------------ exact sigmoids, all outputs
KS = [1, 2, 8, 9, 16, 17, 31, 32, 33, 63, 64, 65, 100, 127, 128, "dense"]


@pytest.fixture(scope="module", params=sorted(SCENES))
def bare(request):
    r = _renderer(SCENES[request.param])
    yield request.param, r
    r.close()


def _exact_inputs(rng, M):
    logits = rng.choice(np.array([-200.0, 0.0, 200.0], F32), (M, 4))
    zp = np.where(rng.random(M) < 0.4, rng.choice(np.array([0.0, 1.0, 2.0, -0.75, 0.5, 1.5, -0.0], F32), M),
                  (rng.standard_normal(M) * 1.5).astype(F32)).astype(F32)
    z = (rng.standard_normal(M) * 10.0 ** rng.integers(-3, 4, M)).astype(F32)
    z[rng.random(M) < 0.05] = rng.choice(np.array([0.0, -0.0], F32))          # live samples at z = +-0
    return logits, zp, z


@pytest.mark.parametrize("K", KS)
def test_all_outputs_with_exact_sigmoids(bare, K):
    """K <= 32: the thread kernel, K > 32: the warp kernel, "dense": the warp kernel with dense = 1 (zp = raw0 rows, z
    from the dense table).  Logits in {-200, 0, 200} make every sigmoid exact; zp and z are arbitrary fp32 values."""
    name, r = bare
    scene = SCENES[name]
    rng = np.random.default_rng([len(name), 0 if K == "dense" else K])
    if K == "dense":
        n = 300
        logits, zp, _ = _exact_inputs(rng, n * 128)
        zp[:128 * 4] = 0.0                                   # rays with acc = 0
        out = _stage5(r, logits, zp.reshape(n, 128), None, None, None, 128, dense=True)
        emu = se.stage5_dense(_sig64(logits).astype(F32), zp.reshape(n, 128), se.zlut_dense(scene, 128))
    else:
        off, cnt = _layout(K, rng)
        logits, zp, z = _exact_inputs(rng, int(cnt.sum()))
        out = _stage5(r, logits, zp, z, off, cnt, K)
        emu = se.stage5(_sig64(logits).astype(F32), zp, z, off, cnt, K)
    n_clamped = _check_all(out, emu, scene, f"{name} K={K}")
    assert np.isnan(se.disp_map(emu["depth_map"], emu["acc_map"])).any()                 # rays with acc = 0
    if not scene.get("use_ndc"):
        assert n_clamped > 0


def _one_sample(values_zp, values_z, logit_a=200.0):
    """One sample per ray with every sigmoid 1 (logit 200): alpha = w = rgb = acc = zp and depth_map = zp z exactly."""
    n = len(values_zp)
    logits = np.full((n, 4), 200.0, F32)
    logits[:, 3] = logit_a
    return logits, np.asarray(values_zp, F32), np.asarray(values_z, F32), np.arange(n, dtype=np.int32), np.ones(n, np.int32)


def test_chosen_per_ray_values():
    """rgba8 through NaN, +-inf, +-0, k/255 +- 1 ulp and 1 - ulp; disp_map and depth_est through acc = 0 (logit -200, zp =
    0, count 0), dm / acc = +-inf and NaN, negative acc, and dm - dr_min < 0, = 0 and denormal (a scene with dr_min = 0)."""
    ks = (np.arange(256, dtype=F64) / 255.0).astype(F32)
    pix = np.concatenate([np.array([np.nan, np.inf, -np.inf, 0.0, -0.0, 1.0, np.nextafter(F32(1), F32(0)), 2.0, -1.0], F32),
                          ks, np.nextafter(ks, F32(2)), np.nextafter(ks, F32(-1))]).astype(F32)
    den = F32(2.0 ** -140)
    for scene in (dict(orc.SCENE_BARBERSHOP), dict(orc.SCENE_BARBERSHOP, depth_range=[0.0, 7.0])):
        dr0 = F32(scene["depth_range"][0])
        r = _renderer(scene)
        zp = [1.0, 1.0, 1.0, 1.0, 1e-30, -0.5, -0.5, 2.0 ** -140, 1.0, 1.0, 0.0, np.inf]
        z = [dr0, np.nextafter(dr0, F32(1)), np.nextafter(dr0, F32(-1)), den, 1e30, -3.0, 3.0, 1e30, np.inf, -np.inf, 5.0, 0.0]
        logits, zp, z, off, cnt = _one_sample(np.concatenate([zp, pix]), np.concatenate([z, np.ones(len(pix), F32)]))
        lg0, zp0, z0, _, _ = _one_sample([1.0, 0.0], [2.0, 2.0], logit_a=-200.0)           # acc = 0 by the logit / zp
        logits, zp, z = np.concatenate([logits, lg0]), np.concatenate([zp, zp0]), np.concatenate([z, z0])
        cnt = np.concatenate([cnt, [1, 1, 0]]).astype(np.int32)                              # ... and by count 0
        off = np.concatenate([off, [len(off), len(off) + 1, len(off) + 2]]).astype(np.int32)
        for K in (4, 40):                                                                    # thread and warp kernel
            out = _stage5(r, logits, zp, z, off, cnt, K)
            emu = se.stage5(_sig64(logits).astype(F32), zp, z, off, cnt, K)
            _check_all(out, emu, scene, f"dr0 {dr0} K={K}")
            o = {k: v.cpu().numpy() for k, v in out.items()}
            p = o["rgba8"][12:12 + len(pix)]
            # NaN -> 0 (the saturate nvcc makes of the viewer's clamp), -inf -> 0, 1 - ulp -> 254; +inf -> 255 in the
            # thread kernel, while in the warp kernel lanes 1..31 add 0 * inf = NaN to it (-> 0)
            assert p[0, 0] == 0 and p[1, 0] == (255 if K <= 32 else 0) and p[2, 0] == 0 and p[3, 0] == 0 and p[6, 0] == 254
            assert (p[:, 3] == 255).all()
            assert np.isnan(o["disp_map"][-3:]).all() and (o["acc_map"][-3:] == 0).all()
            assert o["disp_map"][8] == 0 and o["disp_map"][9] == F32(1e10) and o["disp_map"][5] == F32(1e10)
            assert np.isnan(o["z_vals"][11, 0]) and o["z_vals"][10, 0] == F32(5.0)
        r.close()


@pytest.mark.parametrize("K", [8, 17, 32, 33, 64, 128])
def test_general_logits(K):
    """alpha and acc_map within _composite_f64's operation-count bound; disp_map, rgba8 bit for bit and depth_est within
    its bound as functions of the kernel's own depth_map / acc_map / rgb."""
    scene = orc.SCENE_BARBERSHOP
    r = _renderer(scene)
    rng = np.random.default_rng(200 + K)
    off, cnt = _layout(K, rng, n_random=2000)
    M = int(cnt.sum())
    logits = np.clip(rng.standard_normal((M, 4)) * 4, -16, 16).astype(F32)
    logits[: M // 8, :3] *= 0.25                                            # rgb near 0.5, across many pixel levels
    zp, z = rng.uniform(0, 1.2, M).astype(F32), rng.uniform(0, 10, M).astype(F32)      # _composite_f64 needs z >= 0
    out = _stage5(r, logits, zp, z, off, cnt, K)
    ref, bound = _composite_f64(logits, zp.astype(F64), z.astype(F64), off, cnt, K)
    o = {k: v.cpu().numpy() for k, v in out.items()}
    for k in ("rgb", "weights", "alpha", "depth_map", "acc_map"):
        err = np.abs(o[k].astype(F64) - ref[k])
        assert (err <= bound[k]).all(), f"K={K} {k}: {(err / np.maximum(bound[k], 1e-300)).max():.3f} x bound"
    _check_epilogue(o, scene, f"K={K}")
    assert len(np.unique(o["rgba8"][:, :3])) > 100
    r.close()


# ------------------------------------------------------------------------------------------------ through the driver
def _zero_cell_scene(cell=40):
    """Barbershop with depth_range[0] = -(w_cell - 1), so that the adaptive table's cell `cell` is exactly 0 (the
    reference then stores NaN for every live sample there).  dr1 keeps dr1 - dr0; a few rounds reach the fixed point."""
    scene = dict(orc.SCENE_BARBERSHOP)
    dr0, dr1 = (float(F32(v)) for v in scene["depth_range"])
    span = dr1 - dr0
    zc = float((F32(cell) + F32(0.5)) * F32(1.0 / 128.0))
    for _ in range(20):
        w = F32(math.pow((dr1 - dr0) + 1.0, zc))
        dr0 = float(-(w - F32(1)))
        dr1 = float(F32(dr0 + span))
        scene["depth_range"] = [dr0, dr1]
        if se.zlut(scene)[cell] == 0:
            return scene
    raise AssertionError("no depth range with a zero cell found")


def _zero_alpha(sd1):
    """A shading net whose alpha logit is exactly -200: zero alpha_linear weights, bias -200."""
    sd = {k: v.clone() for k, v in sd1.items()}
    sd["alpha_linear.weight"].zero_()
    sd["alpha_linear.bias"].fill_(-200.0)
    return sd


W, H = 320, 200
DRIVER = {   # name: (scene, shading-net transform, thr, K, sample budget per ray)
    "k8": (orc.SCENE_BARBERSHOP, None, 0.2, 8, 0),
    "k48": (orc.SCENE_BARBERSHOP, None, 0.15, 48, 0),
    "dense": (orc.SCENE_BARBERSHOP, None, 0.0, 128, 0),
    "budget": (orc.SCENE_BARBERSHOP, None, 0.05, 16, 5),
    "zero_alpha": (orc.SCENE_PAVILLON, _zero_alpha, 0.2, 8, 0),
    "zero_cell": ("zero_cell", None, 0.2, 16, 0),
}


def _compose(r, scene, pose, rot, dirs, thr, K):
    """Every stage-5 output of the frame from the stage entry points: stage 0 -> mlp0 -> stage 2 (or the dense table)
    -> stage 3 -> mlp1 -> adn_stage5_composite_aux."""
    x0, ro, rd = r.stage0(pose, rot, dirs)
    raw0 = r.mlp0(x0)
    n = dirs.shape[0]
    if thr == 0.0:
        z = torch.from_numpy(np.tile(se.zlut_dense(scene, 128), n)).cuda()
        ray = torch.arange(n, dtype=torch.int32, device="cuda").repeat_interleave(128)
        raw1 = r.mlp1(r.stage3(ro, rd, ray, z))
        return r.stage5(raw1, raw0, None, None, None, 128, aux=True, dense=True, rgba8=True, out=_prefilled(n, K)), None
    s2 = r.stage2(raw0, thr, K)
    raw1 = r.mlp1(r.stage3(ro, rd, s2["ray"], s2["z"]))
    return r.stage5(raw1, s2["zp"], s2["z"], s2["offset"], s2["count"], K, aux=True, rgba8=True, out=_prefilled(n, K)), s2


def _bits_equal(a, b, what):
    if a.dtype == torch.float32:
        a, b = a.view(torch.int32), b.view(torch.int32)
    assert torch.equal(a, b), what


@pytest.mark.parametrize("case", sorted(DRIVER))
def test_render_entry_points_equal_the_composed_stages(case):
    """render_rays(want_aux=True) and render_camera_rgba8, whole frame and a row band, with chunk_rays unset, 1000 (1024:
    a partial last chunk; whole rows for the camera) -- every aux output, rgb and the pixels equal adn_stage5_composite_aux
    on the composed stages, bit for bit, on pre-filled buffers."""
    scene, tf, thr, K, per_ray = DRIVER[case]
    sd0, sd1 = orc.make_weights("shaped", seed=0)
    pose, rot = torch.tensor(orc.SCENE_BARBERSHOP["view_cell_center"]), orc.rotation_yaw(25.0)
    if scene == "zero_cell":     # put the frame's most selected cell at z = 0 (raw0 does not depend on the depth range)
        r = _renderer(orc.SCENE_BARBERSHOP, sd0, sd1)
        cells = r.stage2(r.mlp0(r.stage0(pose, rot, r.generate_ray_directions(W, H))[0]), thr, K)["cell"]
        scene = _zero_cell_scene(int(torch.bincount(cells.long()).argmax()))
        r.close()
    r = _renderer(scene, sd0, tf(sd1) if tf else sd1)
    pose = torch.tensor(scene["view_cell_center"])
    dirs = r.generate_ray_directions(W, H)
    n = W * H
    for chunk in (0, 1000):
        r.set_option("chunk_rays", chunk)
        for row0, rows in ((0, H), (37, 51)):
            band = slice(row0 * W, (row0 + rows) * W)
            m = rows * W
            if per_ray:
                r.set_option("sample_budget", per_ray * m)
            buf = _prefilled(m, K)
            got = r.render_rays(pose, rot, dirs[band].contiguous(), thr, K, want_aux=True, out=buf["rgb"], aux_out=buf)
            px = r.render_camera_rgba8(pose, rot, W, H, thr, K, row0=row0, rows=rows, out=_filled((m, 4), torch.uint8))
            t = r.last_threshold() if per_ray else thr
            if per_ray:
                r.set_option("sample_budget", 0)
                assert t > thr
            want, s2 = _compose(r, scene, pose, rot, dirs[band].contiguous(), t, K)
            tag = f"{case} chunk {chunk} rows {row0}+{rows}"
            for k in ("rgb",) + AUX:
                _bits_equal(got[k], want[k], f"{tag}: {k}")
            _bits_equal(px, want["rgba8"], f"{tag}: rgba8")
            if chunk and row0 == 0:
                assert n % 1024 and n > 2 * 1024
    o = {k: v.cpu().numpy() for k, v in want.items()}
    if case == "zero_alpha":
        assert (o["acc_map"] == 0).all() and np.isnan(o["disp_map"]).all() and (o["rgba8"][:, :3] == 0).all()
    if case == "zero_cell":
        live = np.arange(K)[None, :] < s2["count"].cpu().numpy()[:, None]
        zero = np.zeros_like(live)
        zero[live] = s2["z"].cpu().numpy() == 0
        assert zero.sum() > 100
        np.testing.assert_array_equal(np.isnan(o["z_vals"]), ~live | zero)
    r.close()
