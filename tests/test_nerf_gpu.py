"""Plain NeRF on the device (option "sampler" = 2, rayMarchSampler LinearlySpacedZNearZFar): the ray kernel and the depth
table bit for bit, every render entry against the stage entries composed by hand, end to end against the reference's
fixtures (tests/golden/nerf_*.npz), the refusals and the export-directory path through the headless viewer."""
import json
import os
import subprocess

import numpy as np
import pytest
import torch

from adanerf_b200 import Renderer
from adanerf_b200 import onnx_weights as ow
from adanerf_b200.synthetic import load_npz
from oracle import adanerf_oracle as orc
from oracle import nerf_oracle as nfo
from oracle import nerf_emulation as nem
from oracle import stage_emulation as em
from oracle.gen_nerf_golden import CASES, case_inputs

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
AUX = Renderer.AUX_KEYS
# bounds set from the H100 run (DESIGN §4.9), with margin: PSNR over the rays whose densities kept their sign under bf16
# (59.1 dB measured at worst), the share of such sign flips on the trained net (17.6 % at worst)
PSNR_KEPT_MIN = 55.0
FLIPPED_MAX_TRAINED = 0.25


@pytest.fixture(scope="module", autouse=True)
def built():
    import __graft_entry__ as g
    g.build()


def _renderer(scene, sd):
    r = Renderer(scene, shading_net=sd)
    r.set_option("sampler", 2)
    return r


def _scene(space):
    return dict(orc.SCENE_PAVILLON_NDC) if space == "ndc" else dict(orc.SCENE_PAVILLON)


@pytest.mark.parametrize("space", ["world", "ndc"])
def test_camera_rays_bit_exact_full_frame(space):
    scene, sd = _scene(space), orc.make_weights("rand", seed=1)[1]
    r = _renderer(scene, sd)
    dirs = r.generate_ray_directions(800, 800)
    pose = torch.tensor(scene["view_cell_center"]) + torch.tensor([0.03, -0.02, 0.01])
    rot = orc.rotation_yaw(37.0)
    out = r.camera_rays(pose, rot, dirs)
    torch.cuda.synchronize()
    o, d, v = nem.camera_rays(pose.numpy(), rot.numpy(), dirs.cpu().numpy(), scene)
    np.testing.assert_array_equal(out["ray_o"].cpu().numpy(), o)
    np.testing.assert_array_equal(out["ray_d"].cpu().numpy(), d)
    np.testing.assert_array_equal(out["ray_dirs"].cpu().numpy(), v)


@pytest.mark.parametrize("space", ["world", "ndc"])
def test_linear_depths_equal_the_table_and_torch(space):
    """Every K: the host table's bits (stage_emulation.zlut_dense); against torch's depths equal on NDC scenes and within
    two ulps of w = base^z on world scenes (tests/test_nerf_oracle.py::test_depth_table_against_torch)."""
    scene = _scene(space)
    r = _renderer(scene, orc.make_weights("rand", seed=1)[1])
    for K in range(1, 129):
        z = r.linear_depths(K).cpu().numpy()
        np.testing.assert_array_equal(z, em.zlut_dense(scene, K))
        t = nfo.linear_depths(K, scene).numpy()[0]
        if space == "ndc":
            np.testing.assert_array_equal(z, t)
        else:
            w = (z - np.float32(scene["depth_range"][0])) + np.float32(1)
            assert (np.abs(z.astype(np.float64) - t) <= 2 * np.spacing(w)).all()


def _by_hand(r, pose, rot, dirs, K):
    """adn_camera_rays -> adn_linear_depths -> adn_stage3_encode -> adn_mlp1_forward -> adn_stage5_density_composite."""
    n = dirs.shape[0]
    rays = r.camera_rays(pose, rot, dirs)
    z = r.linear_depths(K).repeat(n)
    ray_idx = torch.arange(n, device=z.device, dtype=torch.int32).repeat_interleave(K)
    raw1 = r.mlp1(r.stage3(rays["ray_o"], rays["ray_d"], ray_idx, z))
    out = r.stage5_density(raw1, z, rays["ray_dirs"], K, aux=True, rgba8=True)
    out["raw1"] = raw1
    return out


@pytest.mark.parametrize("space,K", [("world", 1), ("world", 7), ("world", 64), ("ndc", 33), ("ndc", 128)])
def test_render_entries_equal_the_stages_by_hand(space, K):
    scene = dict(_scene(space))
    sd = orc.make_weights("rand", seed=2)[1]
    W, H = 160, 96
    r = _renderer(scene, sd)
    pose = torch.tensor(scene["view_cell_center"]) + torch.tensor([0.02, 0.01, -0.03])
    rot = orc.rotation_yaw(11.0)
    dirs = r.generate_ray_directions(W, H)
    ref = _by_hand(r, pose, rot, dirs, K)
    torch.cuda.synchronize()
    for chunk in (0, 1000):
        r.set_option("chunk_rays", chunk)
        out = r.render_rays(pose, rot, dirs, 0.0, K, want_aux=True)
        torch.cuda.synchronize()
        for k in ("rgb",) + AUX:
            np.testing.assert_array_equal(out[k].cpu().numpy(), ref[k].cpu().numpy(), err_msg=f"{k} chunk {chunk}")
        assert (out["n_samples"] == K).all()
        assert not torch.isnan(out["z_vals"]).any()
        host = r.render_rays_host(pose, rot, dirs.cpu().numpy(), 0.0, K)
        np.testing.assert_array_equal(host["rgb"], ref["rgb"].cpu().numpy())
        assert (host["n_samples"] == K).all()
        if space == "world":   # camera entries: the frame's own pinhole rays (NDC projection from the frame, as the viewer)
            cam = r.render_camera(pose, rot, W, H, 0.0, K, want_nsamples=True)
            rgba = r.render_camera_rgba8(pose, rot, W, H, 0.0, K)
            camh = r.render_camera_host(pose, rot, W, H, 0.0, K)
            torch.cuda.synchronize()
            np.testing.assert_array_equal(cam["rgb"].cpu().numpy(), ref["rgb"].cpu().numpy())
            np.testing.assert_array_equal(rgba.cpu().numpy(), ref["rgba8"].cpu().numpy())
            np.testing.assert_array_equal(camh["rgb"], ref["rgb"].cpu().numpy())
    r.set_option("chunk_rays", 0)
    r.set_option("profile", 1)
    r.render_rays(pose, rot, dirs, 0.0, K)
    st = r.stats()
    assert st["n_samples"] == W * H * K and st["ms_stage"][1] == 0.0 and st["ms_stage"][4] > 0.0


def test_options_are_validated():
    """The option checks on a two-network context: pdf_transform 0, sampler 3, and sampler 2 (one network only) are refused;
    a budget under the fixed-K sampler is refused; sampling_view still draws the sampling net's view under sampler 1."""
    from adanerf_b200._lib import AdnError
    from adanerf_b200.synthetic import load_weights_npz
    sd0, sd1 = load_weights_npz(os.path.join(GOLDEN, "weights_pavillon"))
    scene = orc.SCENE_PAVILLON
    r = Renderer(scene, sampling_net=sd0, shading_net=sd1)
    r.set_option("sampler", 1)
    with pytest.raises(AdnError, match="pdf_transform"):
        r.set_option("pdf_transform", 0)
    with pytest.raises(AdnError, match="sampler must be"):
        r.set_option("sampler", 3)
    with pytest.raises(AdnError, match="holds a sampling network"):
        r.set_option("sampler", 2)
    r.set_option("sampler", 1)
    dirs = r.generate_ray_directions(16, 16)
    pose = torch.tensor(scene["view_cell_center"])
    r.set_option("sample_budget", 10_000)
    try:
        with pytest.raises(AdnError, match="sample_budget"):
            r.render_rays(pose, torch.eye(3), dirs, 0.5, 8)
    finally:
        r.set_option("sample_budget", 0)
    r.set_option("sampling_view", 1)
    try:
        v = r.render_rays(pose, torch.eye(3), dirs, 0.5, 8, want_oracle_weights=True)
        assert torch.equal(v["rgb"], r.sampling_view(v["oracle_weights"], rgba8=False)["rgb"])
    finally:
        r.set_option("sampling_view", 0)
    r.close()


def test_refusals():
    scene, sd = _scene("world"), orc.make_weights("rand", seed=1)[1]
    r = _renderer(scene, sd)
    dirs = r.generate_ray_directions(32, 32)
    pose, rot = torch.tensor(scene["view_cell_center"]), torch.eye(3)
    from adanerf_b200._lib import AdnError
    with pytest.raises(AdnError, match="d_oracle_weights"):
        r.render_rays(pose, rot, dirs, 0.0, 8, want_oracle_weights=True)
    r.set_option("sample_budget", 10_000)
    with pytest.raises(AdnError, match="sample_budget"):
        r.render_rays(pose, rot, dirs, 0.0, 8)
    r.set_option("sample_budget", 0)
    r.set_option("sampling_view", 1)
    with pytest.raises(AdnError, match="sampling_view"):
        r.render_rays(pose, rot, dirs, 0.0, 8)
    r.set_option("sampling_view", 0)
    for K in (0, 129):
        with pytest.raises(AdnError):
            r.render_rays(pose, rot, dirs, 0.0, K)
    with pytest.raises(AdnError):
        r.set_option("sampler", 3)
    with pytest.raises(AdnError, match="no sampling network"):   # a one-network context takes no sampling net
        r.set_weights(0, orc.make_weights("rand", seed=1)[0])
    r.render_rays(pose, rot, dirs, 0.0, 8)   # still renders after the refusals
    r.set_option("sampler", 0)
    r.set_weights(0, orc.make_weights("rand", seed=1)[0])   # back to a two-network context: the sampling slot takes a net
    with pytest.raises(AdnError, match="holds a sampling network"):
        r.set_option("sampler", 2)


def _psnr(a, b):
    return 10.0 * np.log10(1.0 / np.mean((np.asarray(a, np.float64) - np.asarray(b, np.float64)) ** 2))


@pytest.mark.parametrize("i", range(len(CASES)), ids=[f"{n}-{s}-k{k}" for n, s, k in CASES])
def test_end_to_end_against_fixtures(i):
    """The device against the reference's fixture: PSNR over all rays and over the rays whose densities kept their sign
    under the MLP's bf16 rounding, and |dPSNR| against a common reference (the float64 oracle plus fixed noise of sigma
    0.03, a ~30 dB image): the project's parity bar is |dPSNR| < 0.05 dB.  It holds over all rays on the trained net and
    over the kept rays everywhere; on the random nets a density near 0 whose sign flips changes a whole ray (the last
    sample's distance is 1e10), which moved up to 39 % of the rays and 4.2 dB on the H100."""
    nets, space, K = CASES[i]
    g = load_npz(os.path.join(GOLDEN, f"nerf_{nets}_{space}_k{K}.npz"))
    scene, pose, rot, dirs, sd = case_inputs(nets, space, 300 + i)
    r = _renderer(scene, sd)
    out = r.render_rays(pose, rot, dirs.cuda(), 0.0, K, want_aux=True)
    hand = _by_hand(r, pose, rot, dirs.cuda(), K)
    torch.cuda.synchronize()
    rgb = out["rgb"].cpu().numpy()
    np.testing.assert_array_equal(rgb, hand["rgb"].cpu().numpy())
    a_dev = hand["raw1"].cpu().numpy().reshape(-1, K, 4)[..., 3]
    flipped = ((a_dev > 0) != (g["raw1"][..., 3] > 0)).any(1)
    kept = ~flipped
    p_all = _psnr(rgb, g["rgb"]) if not np.array_equal(rgb, g["rgb"]) else np.inf
    p_kept = _psnr(rgb[kept], g["rgb"][kept]) if kept.any() and not np.array_equal(rgb[kept], g["rgb"][kept]) else np.inf
    o64 = nfo.render_rays(pose.double(), rot.double(), dirs.double(), orc.to_dtype(sd, torch.float64), scene, K)["rgb"].numpy()
    common = o64 + np.random.default_rng(i).normal(0.0, 0.03, o64.shape)
    d_psnr = _psnr(rgb, common) - _psnr(g["rgb"], common)
    d_kept = _psnr(rgb[kept], common[kept]) - _psnr(g["rgb"][kept], common[kept]) if kept.any() else 0.0
    print(json.dumps(dict(case=f"{nets}-{space}-k{K}", psnr_all=round(float(p_all), 2), psnr_kept=round(float(p_kept), 2),
                          flipped_rays=int(flipped.sum()), n_rays=int(len(rgb)), d_psnr=round(float(d_psnr), 5),
                          d_psnr_kept=round(float(d_kept), 5))))
    assert abs(d_kept) < 0.05
    assert p_kept >= PSNR_KEPT_MIN
    if nets == "pav":
        assert abs(d_psnr) < 0.05 and flipped.mean() <= FLIPPED_MAX_TRAINED
    np.testing.assert_allclose(out["z_vals"].cpu().numpy(), g["z"], rtol=0, atol=2e-6 * max(1.0, float(np.abs(g["z"]).max())))
    if K == 1:
        assert not rgb.any()


def test_headless_viewer_renders_converted_export(tmp_path):
    from adanerf_b200 import convert
    sd = orc.make_weights("rand", seed=5)[1]
    torch.save(sd, tmp_path / "Net0_opt.weights")
    scene = orc.SCENE_PAVILLON
    with open(tmp_path / "dataset_info.txt", "w") as f:
        for k in ("view_cell_center", "view_cell_size", "depth_range", "fov", "max_depth"):
            f.write(f"{k} = {scene[k]}\n")
    out = tmp_path / "nerf"
    convert.main(["--weights0", str(tmp_path / "Net0_opt.weights"), "--dataset-info", str(tmp_path / "dataset_info.txt"),
                  "--samples", "32", "--out", str(out), "--sampler", "LinearlySpacedZNearZFar"])
    viewer = os.path.join(ROOT, "adanerf_b200", "adn_viewer_headless")
    p = subprocess.run([viewer, str(out), "-s", "96", "64", "-f", "2"], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stdout + p.stderr
    assert "checksum" in p.stdout
    p = subprocess.run([viewer, str(out), "-s", "96", "64", "-f", "1", "--oracle"], capture_output=True, text=True, timeout=300)
    assert p.returncode == 2 and "one-network export" in p.stderr
    r, thr, k = Renderer.from_export_dir(str(out))
    assert k == 32
    img = r.render_camera(torch.tensor(scene["view_cell_center"]), torch.eye(3), 96, 64, 0.0, k)["rgb"]
    torch.cuda.synchronize()
    assert torch.isfinite(img).all()


def test_two_gpu_bands_equal_one_gpu():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    from adanerf_b200.multi import MultiRenderer
    scene, sd = _scene("world"), orc.make_weights("rand", seed=1)[1]
    pose, rot = torch.tensor(scene["view_cell_center"]), orc.rotation_yaw(5.0)
    one = _renderer(scene, sd).render_camera(pose, rot, 128, 96, 0.0, 16)["rgb"].cpu().numpy()
    m = MultiRenderer(scene, [0, 1], shading_net=sd)
    m.set_option("sampler", 2)
    m.render_camera(pose, rot, 128, 96, 0.0, 16)
    two = m.wait_frame()
    np.testing.assert_array_equal(two.cpu().numpy().reshape(one.shape), one)
