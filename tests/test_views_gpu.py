"""Several cameras in one call on the device (adn_render_views_rays / _camera / _camera_rgba8, Renderer.render_views,
B200Inference on an n_images > 1 batch, the headless viewer's --views): bit for bit the single-view calls concatenated, for
every sampler, world and NDC scenes, dense mode, every aux output, OracleWeights, RGBA8 and sampling_view, across chunk
boundaries inside a view; one threshold under one sample budget; the refusals."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest
import torch

from adanerf_b200 import AdnError, Renderer
from oracle import adanerf_oracle as orc

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
AUX = Renderer.AUX_KEYS
ADN_ERR_INVALID = 1


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as g
    g.build()
    return g


def _cameras(scene, V, seed=0):
    """V cameras that differ in position and rotation."""
    g = torch.Generator().manual_seed(seed)
    c = torch.tensor(scene["view_cell_center"], dtype=torch.float32)
    poses = torch.stack([c + 0.05 * torch.randn(3, generator=g) for _ in range(V)])
    rots = torch.stack([orc.rotation_yaw(17.0 + 41.0 * v + seed) for v in range(V)])
    return poses, rots


def _dirs(r, V, N, seed=0):
    """[V, N, 3]: a different random subset of the frame's pixel directions per view."""
    g = torch.Generator().manual_seed(100 + seed)
    d = r.generate_ray_directions(800, 800).cpu()
    return torch.stack([d[torch.randperm(d.shape[0], generator=g)[:N]] for _ in range(V)]).cuda()


# name -> (scene, sampler, thr, K)
CASES = {
    "adaptive_world": (orc.SCENE_PAVILLON, 0, 0.2, 16),
    "adaptive_ndc": (orc.SCENE_PAVILLON_NDC, 0, 0.2, 16),
    "dense_world": (orc.SCENE_PAVILLON, 0, 0.0, 128),
    "donerf_world": (orc.SCENE_PAVILLON, 1, 0.0, 8),
    "nerf_world": (orc.SCENE_PAVILLON, 2, 0.0, 32),
    "nerf_ndc": (orc.SCENE_PAVILLON_NDC, 2, 0.0, 32),
}


def _renderer(case, pavillon_weights):
    """The shipped Pavillon pair; on NDC scenes a pair with the 30-feature sampling net of the NDC configs."""
    scene, sampler, _, _ = CASES[case]
    sd0, sd1 = orc.make_weights("ndc", seed=0) if scene.get("use_ndc") and sampler != 2 else pavillon_weights
    if sampler == 2:
        r = Renderer(scene, shading_net=sd1)
    else:
        r = Renderer(scene, sampling_net=sd0, shading_net=sd1)
    if sampler:
        r.set_option("sampler", sampler)
    return r


def _assert_same(a, b, what):
    a, b = a.cpu().numpy(), b.cpu().numpy()
    assert a.shape == b.shape, what
    np.testing.assert_array_equal(a.view(np.uint8), b.view(np.uint8), err_msg=what)


@pytest.mark.parametrize("chunk", [0, 384], ids=["one_chunk", "chunk_splits_views"])
@pytest.mark.parametrize("V,N", [(1, 1000), (2, 1000), (3, 777)])
@pytest.mark.parametrize("case", sorted(CASES))
def test_views_rays_equal_single_view_calls(pavillon_weights, case, V, N, chunk):
    scene, sampler, thr, K = CASES[case]
    r = _renderer(case, pavillon_weights)
    r.set_option("chunk_rays", chunk)
    poses, rots = _cameras(scene, V, seed=V)
    dirs = _dirs(r, V, N, seed=V)
    ow = sampler != 2
    got = r.render_views(poses, rots, dirs, thr, K, want_oracle_weights=ow, want_aux=True)
    m_views = r.stats()["n_samples"]
    m_single = 0
    for v in range(V):
        want = r.render_rays(poses[v], rots[v], dirs[v], thr, K, want_oracle_weights=ow, want_aux=True)
        m_single += r.stats()["n_samples"]
        for k in ("rgb", "n_samples", "oracle_weights") + AUX:
            if want[k] is not None:
                _assert_same(got[k][v * N:(v + 1) * N], want[k], f"{case} view {v} {k}")
    if chunk == 0:   # adn_get_stats counts the last chunk's samples; one chunk per call here
        assert m_views == m_single
    r.close()


@pytest.mark.parametrize("case", ["adaptive_world", "adaptive_ndc", "donerf_world"])
def test_views_sampling_view_equals_single_view_calls(pavillon_weights, case):
    scene, _, thr, K = CASES[case]
    r = _renderer(case, pavillon_weights)
    r.set_option("sampling_view", 1)
    poses, rots = _cameras(scene, 2, seed=5)
    dirs = _dirs(r, 2, 1000, seed=5)
    got = r.render_views(poses, rots, dirs, thr, K, want_oracle_weights=True)
    for v in range(2):
        want = r.render_rays(poses[v], rots[v], dirs[v], thr, K, want_oracle_weights=True)
        for k in ("rgb", "n_samples", "oracle_weights"):
            _assert_same(got[k][v * 1000:(v + 1) * 1000], want[k], f"view {v} {k}")
    r.close()


@pytest.mark.parametrize("chunk", [0, 3000], ids=["auto_chunk", "chunk_splits_views"])
@pytest.mark.parametrize("case", ["adaptive_world", "adaptive_ndc", "donerf_world", "nerf_world", "nerf_ndc"])
def test_views_camera_equals_single_camera_calls(pavillon_weights, case, chunk):
    """Whole frames generated on the device (ray id -> view, row, column), fp32 and RGBA8; W = 130 is not a multiple of
    128 and a 3000-ray chunk ends inside a row and inside a view."""
    scene, _, thr, K = CASES[case]
    W, H, V = 130, 97, 3
    r = _renderer(case, pavillon_weights)
    r.set_option("chunk_rays", chunk)
    poses, rots = _cameras(scene, V, seed=7)
    got = r.render_views_camera(poses, rots, W, H, thr, K, want_nsamples=True)
    px = r.render_views_camera(poses, rots, W, H, thr, K, rgba8=True)
    n = W * H
    for v in range(V):
        want = r.render_camera(poses[v], rots[v], W, H, thr, K, want_nsamples=True)
        _assert_same(got["rgb"][v * n:(v + 1) * n], want["rgb"], f"view {v} rgb")
        _assert_same(got["n_samples"][v * n:(v + 1) * n], want["n_samples"], f"view {v} n_samples")
        _assert_same(px[v * n:(v + 1) * n], r.render_camera_rgba8(poses[v], rots[v], W, H, thr, K), f"view {v} rgba8")
    r.close()


@pytest.mark.parametrize("chunk", [0, 5000], ids=["one_chunk", "chunk_splits_views"])
def test_stereo_budget_one_threshold(pavillon_weights, chunk):
    """A stereo pair under one B: M <= B over both eyes, one t*, and the call equals the fixed-threshold views call and the
    two single-view calls at that t*."""
    scene, _, thr, K = CASES["adaptive_world"]
    r = _renderer("adaptive_world", pavillon_weights)
    r.set_option("chunk_rays", chunk)
    W = H = 96
    poses, rots = _cameras(scene, 2, seed=11)
    free = r.render_views_camera(poses, rots, W, H, thr, K, want_nsamples=True)
    m_free = int(free["n_samples"].sum())
    B = 2 * W * H + (m_free - 2 * W * H) // 2
    r.set_option("sample_budget", B)
    got = r.render_views_camera(poses, rots, W, H, thr, K, want_nsamples=True)
    t_star = r.last_threshold()
    m = int(got["n_samples"].sum())
    assert m <= B and t_star > thr
    if chunk == 0:
        assert r.stats()["n_samples"] == m
    r.set_option("sample_budget", 0)
    fixed = r.render_views_camera(poses, rots, W, H, t_star, K, want_nsamples=True)
    for k in ("rgb", "n_samples"):
        _assert_same(got[k], fixed[k], k)
    n = W * H
    for v in range(2):
        eye = r.render_camera(poses[v], rots[v], W, H, t_star, K, want_nsamples=True)
        _assert_same(got["rgb"][v * n:(v + 1) * n], eye["rgb"], f"eye {v}")
    # the rays entry under the same budget: one t* over both views, aux outputs included
    dirs = r.generate_ray_directions(W, H).reshape(1, -1, 3).repeat(2, 1, 1)
    r.set_option("sample_budget", B)
    a = r.render_views(poses, rots, dirs, thr, K, want_aux=True, want_oracle_weights=True)
    t2 = r.last_threshold()
    r.set_option("sample_budget", 0)
    b = r.render_views(poses, rots, dirs, t2, K, want_aux=True, want_oracle_weights=True)
    for k in ("rgb", "n_samples", "oracle_weights") + AUX:
        _assert_same(a[k], b[k], k)
    r.close()


def test_views_refusals(pavillon_weights):
    r = _renderer("adaptive_world", pavillon_weights)
    lib, h = r.lib, r.handle
    scene = CASES["adaptive_world"][0]
    poses, rots = _cameras(scene, 65)
    p = np.ascontiguousarray(poses.numpy())
    q = np.ascontiguousarray(rots.numpy().reshape(65, 9))
    fp = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
    dirs = torch.zeros((65 * 4, 3), device="cuda")
    rgb = torch.empty((65 * 4, 3), device="cuda")
    l0 = r.stats()["kernel_launches"]

    def views_rays(V, pp, qq, n, d=dirs.data_ptr(), stream=None):
        return lib.adn_render_views_rays(h, V, pp, qq, d, n, 0.2, 16, rgb.data_ptr(), None, None, None, stream)

    assert views_rays(0, fp(p), fp(q), 4) == ADN_ERR_INVALID
    assert views_rays(65, fp(p), fp(q), 4) == ADN_ERR_INVALID
    assert "1-64" in lib.adn_last_error(h).decode()
    assert views_rays(2, None, fp(q), 4) == ADN_ERR_INVALID
    assert views_rays(2, fp(p), None, 4) == ADN_ERR_INVALID
    assert views_rays(2, fp(p), fp(q), 0) == ADN_ERR_INVALID
    assert views_rays(2, fp(p), fp(q), 4, d=None) == ADN_ERR_INVALID
    assert views_rays(64, fp(p), fp(q), (1 << 62)) == ADN_ERR_INVALID
    assert "overflow" in lib.adn_last_error(h).decode()
    assert lib.adn_render_views_camera(h, 2, fp(p), fp(q), 0, 10, 0.2, 16, rgb.data_ptr(), None, None) == ADN_ERR_INVALID
    assert lib.adn_render_views_camera(h, 64, fp(p), fp(q), 1 << 30, 1 << 30, 0.2, 16, rgb.data_ptr(), None, None) == ADN_ERR_INVALID
    assert lib.adn_render_views_camera_rgba8(h, 0, fp(p), fp(q), 8, 8, 0.2, 16, rgb.data_ptr(), None) == ADN_ERR_INVALID
    # the single-view checks apply to the V N rays: a budget below the call's rays
    r.set_option("sample_budget", 6)
    assert views_rays(2, fp(p), fp(q), 4) == ADN_ERR_INVALID
    r.set_option("sample_budget", 0)
    with pytest.raises(ValueError):
        r.render_views(poses[:2], rots[:3], dirs[:8].reshape(2, 4, 3), 0.2, 16)
    # a capturing stream, with the message of the other entries
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        g.capture_begin()
        try:
            st = views_rays(2, fp(p), fp(q), 4, stream=C.c_void_p(s.cuda_stream))
        finally:
            g.capture_end()
    assert st == ADN_ERR_INVALID and "capturing a CUDA graph" in lib.adn_last_error(h).decode()
    assert r.stats()["kernel_launches"] == l0
    r.close()


def test_adapter_two_image_batch(pavillon_weights):
    """B200Inference.inference on ImagePose [2,3] / RayDirectionsSamples [2,N,3]: the reference's flattened outputs, equal
    to the per-image calls concatenated."""
    from adanerf_b200.adapter import B200Inference, KEY_ASP, KEY_DIRS, KEY_ORACLE, KEY_POSE, KEY_ROT, KEY_DEPTH
    scene = orc.SCENE_PAVILLON
    sd0, sd1 = pavillon_weights
    inf = B200Inference(scene, sd0, sd1, 0.2, 16, want_oracle_weights=True, want_aux=True)
    poses, rots = _cameras(scene, 2, seed=3)
    dirs = _dirs(inf.renderer, 2, 640, seed=3)
    outs, dicts = inf.inference({KEY_POSE: poses, KEY_ROT: rots, KEY_DIRS: dirs})
    assert outs[-1].shape == (1280, 3) and dicts[1][KEY_ASP].shape == (1280,) and dicts[1][KEY_ORACLE].shape == (1280, 128)
    assert dicts[1][KEY_DEPTH].shape == (1280, 1)
    for v in range(2):
        o1, d1 = inf.inference({KEY_POSE: poses[v:v + 1], KEY_ROT: rots[v:v + 1], KEY_DIRS: dirs[v:v + 1]})
        sl = slice(640 * v, 640 * (v + 1))
        _assert_same(outs[-1][sl], o1[-1], f"rgb {v}")
        for k in (KEY_ASP, KEY_ORACLE, KEY_DEPTH):
            _assert_same(dicts[1][k][sl], d1[1][k], f"{k} {v}")
    inf.renderer.close()


def _export(tmp_path, name):
    src = os.path.join(GOLDEN, "shipped", name)
    with open(os.path.join(src, "manifest.json")) as f:
        man = json.load(f)
    for fname, e in man["files"].items():
        data = b""
        for p in e.get("parts", [fname]):
            with open(os.path.join(src, p), "rb") as f:
                data += f.read()
        (tmp_path / fname).write_bytes(data)
    return str(tmp_path)


def test_headless_viewer_views_write_one_ppm_per_view(built, tmp_path):
    """--views 2 -w: two PPMs whose pixels equal single-view renders of the cameras the viewer reports; -g is refused."""
    d = _export(tmp_path, "pavillon_k16")
    W, H = 200, 151
    r = subprocess.run([built.VIEWER, d, "--views", "2", "-s", str(W), str(H), "-f", "3", "-w"], capture_output=True, text=True,
                       timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "x 2 views" in r.stdout, r.stdout
    ren, thr, K = Renderer.from_export_dir(d)
    for v in range(2):
        line = next(l for l in r.stdout.splitlines() if l.startswith(f"view {v}: pos "))
        vals = line.split()
        pose = np.array(vals[3:6], dtype=np.float32)
        rot = np.array(vals[7:16], dtype=np.float32).reshape(3, 3)
        want = ren.render_camera(pose, rot, W, H, thr, K)["rgb"].cpu().numpy().reshape(-1)
        with open(os.path.join(d, f"adn_frame_view{v}.ppm"), "rb") as f:
            data = f.read()
        head = f"P6\n{W} {H}\n255\n".encode()
        assert data.startswith(head)
        px = np.frombuffer(data[len(head):], dtype=np.uint8)
        sat = np.where(want > 0, np.minimum(want, np.float32(1)), np.float32(0)).astype(np.float32)
        np.testing.assert_array_equal(px, (sat * np.float32(255)).astype(np.uint8), err_msg=f"view {v}")
        assert len(set(px.tolist())) > 4
    ren.close()
    bad = subprocess.run([built.VIEWER, d, "--views", "2", "-g", "2"], capture_output=True, text=True, timeout=60)
    assert bad.returncode == 2 and "--views" in bad.stderr


@pytest.mark.parametrize("name", ["pav_k16", "ndc_k16", "donerf_pav_k8", "nerf_pav_k32"])
def test_views_end_to_end_against_reference_fixtures(name):
    """One views call over the fixture's two images against the reference's multi-image inference: |dPSNR| < 0.05 dB against
    a common image (the reference's colours plus fixed noise of sigma 0.03, a ~30 dB image) and, for the adaptive sampler,
    the same sample count on >= 99.9 % of the rays and PSNR >= 49.4 dB against the reference (tests/test_parity_gate.py)."""
    from adanerf_b200.synthetic import load_npz
    from oracle.gen_views_golden import CASES as VCASES, case_inputs
    g = load_npz(os.path.join(GOLDEN, f"views_{name}.npz"))
    sampler, _, K, thr = VCASES[name]
    scene, poses, rots, dirs, sd0, sd1 = case_inputs(name, 500 + list(VCASES).index(name))
    r = Renderer(scene, sampling_net=sd0, shading_net=sd1)
    if sampler:
        r.set_option("sampler", sampler)
    out = r.render_views(poses, rots, dirs.cuda(), thr, K)
    rgb = out["rgb"].cpu().numpy()
    psnr = lambda a, b: 10.0 * np.log10(1.0 / np.mean((np.asarray(a, np.float64) - np.asarray(b, np.float64)) ** 2))
    common = g["rgb"] + np.random.default_rng(0).normal(0.0, 0.03, g["rgb"].shape)
    d_psnr = psnr(rgb, common) - psnr(g["rgb"], common)
    print(json.dumps(dict(case=name, psnr_vs_reference=round(float(psnr(rgb, g["rgb"])), 2), d_psnr=round(float(d_psnr), 5))))
    assert abs(d_psnr) < 0.05
    if sampler == 0:
        same = float(np.mean(out["n_samples"].cpu().numpy() == np.rint(g["asp"] * K).astype(np.int32)))
        assert same >= 0.999 and psnr(rgb, g["rgb"]) >= 49.4
    r.close()
