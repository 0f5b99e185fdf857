"""The fixed-K sampler on the device (option "sampler" = 1, rayMarchSampler FromClassifiedDepth): the inverse-CDF sampler
and the density composite against the CPU oracle (oracle/donerf_oracle.py, pinned to the reference by
tests/golden/donerf_*.npz), end-to-end parity, every render entry point against the stage entries composed by hand, the
multi-GPU frame, the headless viewer, and the adaptive path left as it was."""
import math
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from adanerf_b200 import onnx_weights as ow
from adanerf_b200.synthetic import load_npz, load_weights_npz
from oracle import adanerf_oracle as orc
from oracle import donerf_oracle as dno
from oracle.gen_donerf_golden import CASES

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
TRANSFORM = {"sigmoid": dno.SIGMOID, "softmax": dno.SOFTMAX}


def _renderer(nets, transform=1):
    from adanerf_b200 import Renderer
    if nets == "pav":
        sd0, sd1 = load_weights_npz(os.path.join(GOLDEN, "weights_pavillon"))
        scene = orc.SCENE_PAVILLON
    else:
        sd0, sd1 = orc.make_weights("rand", seed=100)
        scene = orc.SCENE_BARBERSHOP
    r = Renderer(scene, sampling_net=sd0, shading_net=sd1)
    r.set_option("sampler", 1)
    r.set_option("pdf_transform", transform)
    return r, scene, sd0, sd1


@pytest.fixture(scope="module")
def pav():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    r, scene, sd0, sd1 = _renderer("pav")
    yield r, scene, sd0, sd1
    r.close()


def _frame_raw0(r, scene, W, H):
    """raw0 of a W x H frame from the view-cell centre, on the device (stage 0 + the sampling MLP)."""
    dirs = r.generate_ray_directions(W, H)
    pose = torch.tensor(scene["view_cell_center"], dtype=torch.float32)
    x0, ray_o, ray_d = r.stage0(pose, torch.eye(3), dirs)
    return r.mlp0(x0), ray_o, ray_d, dirs, pose


def _to_unit(z, depth_range):
    """World depth -> the sampler's [0, 1] position (LogTransform.from_world without its clamp), in float64."""
    z = np.asarray(z, np.float64)
    return np.log(z - depth_range[0] + 1.0) / math.log(depth_range[1] - depth_range[0] + 1.0)


def _check_z(z_dev, z_ref, depth_range, what):
    """z within 8 ulps of the warped depth on all but 5 % of the samples (the oracle's fp32 sum and softmax denominator are
    ATen's own order; on full frames of the Pavillon networks it is under 0.03 %, on the random networks' flat
    distributions a few %, all within 1e-6 of the warped range), and no further than 1e-5 of the warped range from it on
    all but 0.1 %: those are the samples whose u
    the sampler and the oracle put into different CDF bins next to the denom < 1e-5 clamp, where z may jump by up to one
    depth cell (1/128 of the warped range)."""
    zd, zr = z_dev.reshape(-1).cpu().numpy(), z_ref.reshape(-1).numpy()
    assert np.isfinite(zd).all()
    tol = 8 * np.spacing(np.abs(zr).astype(np.float32)).astype(np.float64)
    err = np.abs(zd.astype(np.float64) - zr)
    du = np.abs(_to_unit(zd, depth_range) - _to_unit(zr, depth_range))
    i = int(np.argmax(err))
    print(f"{what}: worst |dz| {err[i]:.3g} at sample {i} (z {zr[i]:.6g}), {(err > tol).mean() * 100:.4f} % beyond 8 ulp, "
          f"{(du > 1e-5).mean() * 100:.4f} % jumped, largest jump {du.max():.3g} of the warped range")
    assert (err > tol).mean() <= 5e-2, what
    assert (du > 1e-5).mean() <= 1e-3, what
    assert du.max() <= 1.0 / 128 + 1e-6, what


@pytest.mark.parametrize("K", [1, 8, 16, 128])
def test_sampler_matches_oracle_full_frame(pav, K):
    r, scene, _, _ = pav
    raw0, _, _, _, _ = _frame_raw0(r, scene, 800, 800)
    n = raw0.shape[0]
    for transform in (dno.SIGMOID, dno.SOFTMAX):
        s = r.pdf_sample(raw0, K, transform)
        torch.cuda.synchronize()
        ref = dno.pdf_sample(raw0.cpu(), K, transform, scene["depth_range"])
        assert torch.equal(s["count"].cpu(), torch.full((n,), K, dtype=torch.int32))
        assert torch.equal(s["offset"].cpu(), torch.arange(n, dtype=torch.int32) * K)
        assert torch.equal(s["ray"].cpu(), torch.arange(n, dtype=torch.int32).repeat_interleave(K))
        _check_z(s["z"], ref, scene["depth_range"], f"800x800 K={K} transform={transform}")


def test_sampler_partial_tile_and_fixtures(pav):
    """A ray count that leaves the last CTA partly empty, and the reference's own raw0 from every fixture."""
    r, scene, _, _ = pav
    raw0, _, _, _, _ = _frame_raw0(r, scene, 37, 29)   # 1073 rays: 134 CTAs of 8 and one of 1
    s = r.pdf_sample(raw0, 5, dno.SIGMOID)
    ref = dno.pdf_sample(raw0.cpu(), 5, dno.SIGMOID, scene["depth_range"])
    assert torch.equal(s["ray"].cpu(), torch.arange(raw0.shape[0], dtype=torch.int32).repeat_interleave(5))
    _check_z(s["z"], ref, scene["depth_range"], "1073 rays K=5")
    for nets, tname, K in CASES:
        g = load_npz(os.path.join(GOLDEN, f"donerf_{nets}_{tname}_k{K}.npz"))
        dr = (orc.SCENE_PAVILLON if nets == "pav" else orc.SCENE_BARBERSHOP)["depth_range"]
        from adanerf_b200 import Renderer
        rr = Renderer(orc.SCENE_PAVILLON if nets == "pav" else orc.SCENE_BARBERSHOP)
        s = rr.pdf_sample(torch.from_numpy(g["raw0"]), K, TRANSFORM[tname])
        _check_z(s["z"], torch.from_numpy(g["z"]), dr, f"fixture {nets} {tname} K={K}")
        rr.close()


def _composite_close(out, ref, K):
    for k, kr, atol in (("rgb", "rgb", 2e-6), ("weights", "weights", 2e-6), ("alpha", "alpha", 2e-6), ("acc_map", "acc", 4e-6)):
        a, b = out[k].cpu().numpy(), ref[kr].numpy()
        if b.ndim == 2 and b.shape[1] == 0:   # K = 1: the reference's weights / alpha are [N, 0]; ours are [N, 1] of zeros
            b = np.zeros_like(a)
        np.testing.assert_allclose(a, b, rtol=1e-5, atol=atol, err_msg=f"{k} K={K}")
    np.testing.assert_allclose(out["depth_map"].cpu().numpy(), ref["depth_map"].numpy(), rtol=1e-5, atol=1e-5)
    d, dr = out["disp_map"].cpu().numpy(), ref["disp"].numpy()
    assert np.array_equal(np.isnan(d), np.isnan(dr)), "NaN disparity where acc == 0, as the adaptive composite"
    m = ~np.isnan(dr)
    np.testing.assert_allclose(d[m], dr[m], rtol=1e-3)   # depth_map / acc: two sums, in a shuffle tree for K > 32


def test_composite_matches_oracle(pav):
    r, _, _, _ = pav
    # the reference's raw1 / z / rays_d of every fixture (K = 1 .. 16: the thread-per-ray kernel)
    for nets, tname, K in CASES:
        g = load_npz(os.path.join(GOLDEN, f"donerf_{nets}_{tname}_k{K}.npz"))
        n = g["ray_d"].shape[0]
        out = r.stage5_density(torch.from_numpy(g["raw1"].reshape(n * K, 4)), torch.from_numpy(g["z"].reshape(-1)),
                               torch.from_numpy(g["ray_d"]), K)
        ref = dno.nerf_raw2outputs(torch.from_numpy(g["raw1"]), torch.from_numpy(g["z"]), torch.from_numpy(g["ray_d"]))
        np.testing.assert_allclose(out["rgb"].cpu().numpy(), g["rgb"], rtol=1e-5, atol=2e-6)
        _composite_close(out, ref, K)
        np.testing.assert_array_equal(out["z_vals"].cpu().numpy(), g["z"])
    # K = 64 and 128 (the warp-per-ray kernel) on synthetic inputs, with rays whose every alpha is 0 (acc = 0: NaN disp)
    gen = torch.Generator().manual_seed(7)
    for K in (33, 64, 128):
        n = 300
        raw1 = torch.randn(n, K, 4, generator=gen) * 2
        raw1[::7, :, 3] = -5.0
        z = torch.sort(torch.rand(n, K, generator=gen) * 8 + 0.2, dim=1).values
        rd = torch.nn.functional.normalize(torch.randn(n, 3, generator=gen), dim=-1) * 1.0001
        out = r.stage5_density(raw1.reshape(-1, 4), z.reshape(-1), rd, K)
        ref = dno.nerf_raw2outputs(raw1, z, rd)
        _composite_close(out, ref, K)
        assert np.isnan(out["disp_map"].cpu().numpy()[::7]).all()


def _psnr(a, b):
    mse = float(torch.mean((a.double().cpu() - b.double().cpu()) ** 2))
    return float("inf") if mse == 0 else 10 * math.log10(1 / mse)


@pytest.mark.parametrize("i", range(len(CASES)), ids=[f"{n}-{t}-k{k}" for n, t, k in CASES])
def test_end_to_end_against_reference_fixture(i):
    """The whole render against the reference's, on the fixture's rays.  The density composite makes a ray's colour a
    step function of the sign of its densities where they sit near 0 (relu, and the last sample's 1e10 distance), so a
    ray whose bf16 shading net puts any density on the other side of 0 than the reference's fp32 net may change colour
    entirely.  Those rays are counted (at most 8 %: up to 6.3 % measured on the random networks, whose densities sit
    around 0), and the PSNR bound holds on the others: 45 dB (48.7 dB measured at the least, Pavillon K = 4, where the
    wide sample spacing amplifies the bf16 error of the densities); the PSNR over every ray is printed.  Per-ray sample
    counts are exact."""
    from adanerf_b200 import Renderer
    from oracle.gen_donerf_golden import case_inputs
    nets, tname, K = CASES[i]
    g = load_npz(os.path.join(GOLDEN, f"donerf_{nets}_{tname}_k{K}.npz"))
    scene, pose, rot, dirs, sd0, sd1 = case_inputs(nets, 100 + i)
    r = Renderer(scene, sampling_net=sd0, shading_net=sd1)
    r.set_option("sampler", 1)
    r.set_option("pdf_transform", TRANSFORM[tname])
    d = dirs.cuda()
    out = r.render_rays(pose, rot, d, 0.0, K, want_aux=True)
    assert (out["n_samples"].cpu() == K).all()
    assert not torch.isnan(out["z_vals"]).any()
    x0, ray_o, ray_d = r.stage0(pose, rot, d)
    s = r.pdf_sample(r.mlp0(x0), K, TRANSFORM[tname])
    a_dev = r.mlp1(r.stage3(ray_o, ray_d, s["ray"], s["z"]))[:, 3].reshape(-1, K).cpu()
    flip = ((a_dev > 0) != torch.from_numpy(g["raw1"][:, :, 3] > 0)).any(1)
    ref = torch.from_numpy(g["rgb"])
    keep = ~flip
    p_all, p = _psnr(out["rgb"].cpu(), ref), _psnr(out["rgb"].cpu()[keep], ref[keep])
    gt = (ref + 0.05 * torch.randn(ref.shape, generator=torch.Generator().manual_seed(i))).clamp(0, 1)   # a common reference
    dp = abs(_psnr(out["rgb"].cpu()[keep], gt[keep]) - _psnr(ref[keep], gt[keep]))
    print(f"{nets} {tname} K={K}: PSNR(ours, reference) {p_all:.2f} dB over all rays, {p:.2f} dB over the "
          f"{100 * float(keep.float().mean()):.2f} % whose densities keep their sign; |dPSNR| vs a common reference {dp:.4f} dB")
    assert float(flip.float().mean()) <= 0.08
    assert p >= 45.0 and dp < 0.05
    r.close()


def _same(a, b):
    """Bit for bit, NaN included."""
    if a.dtype == torch.float32:
        return torch.equal(a.view(torch.int32), b.view(torch.int32))
    return torch.equal(a, b)


def _compose(r, scene, W, H, K, transform):
    raw0, ray_o, ray_d, dirs, pose = _frame_raw0(r, scene, W, H)
    s = r.pdf_sample(raw0, K, transform)
    raw1 = r.mlp1(r.stage3(ray_o, ray_d, s["ray"], s["z"]))
    out = r.stage5_density(raw1, s["z"], ray_d, K, rgba8=True)
    return out, dirs, pose, raw0


@pytest.mark.parametrize("K", [4, 48])
def test_every_entry_point_equals_the_stages(pav, K):
    r, scene, _, _ = pav
    W, H = 160, 120
    ref, dirs, pose, raw0 = _compose(r, scene, W, H, K, dno.SIGMOID)
    rot = torch.eye(3)
    for fuse in (1, 0):
        r.set_option("fuse_encoder", fuse)
        for chunk in (0, 128 * 13):
            r.set_option("chunk_rays", chunk)
            o = r.render_rays(pose, rot, dirs, 0.5, K, want_oracle_weights=True, want_aux=True)
            assert torch.equal(o["oracle_weights"], raw0)
            for k in ("rgb",) + r.AUX_KEYS:
                assert _same(o[k], ref[k]), (k, fuse, chunk)
            assert (o["n_samples"] == K).all()
            assert torch.equal(r.render_camera(pose, rot, W, H, 0.5, K)["rgb"], ref["rgb"])
            assert torch.equal(r.render_camera_rgba8(pose, rot, W, H, 0.5, K).reshape(-1, 4), ref["rgba8"])
            h = r.render_rays_host(pose, rot, dirs.cpu().numpy(), 0.5, K)
            assert np.array_equal(h["rgb"], ref["rgb"].cpu().numpy()) and (h["n_samples"] == K).all()
            hc = r.render_camera_host(pose, rot, W, H, 0.5, K)
            assert np.array_equal(hc["rgb"], ref["rgb"].cpu().numpy())
    r.set_option("fuse_encoder", 1)
    r.set_option("chunk_rays", 0)
    r.render_camera(pose, rot, W, H, 0.5, K)
    assert r.stats()["n_samples"] == W * H * K   # the samples of the last stage 2: the whole call when it is one chunk


def test_options_are_validated(pav):
    from adanerf_b200 import AdnError
    r, scene, _, _ = pav
    with pytest.raises(AdnError, match="pdf_transform"):
        r.set_option("pdf_transform", 0)
    with pytest.raises(AdnError):
        r.set_option("sampler", 2)
    dirs = r.generate_ray_directions(16, 16)
    pose = torch.tensor(scene["view_cell_center"])
    r.set_option("sample_budget", 10_000)
    try:
        with pytest.raises(AdnError, match="sample_budget"):
            r.render_rays(pose, torch.eye(3), dirs, 0.5, 8)
    finally:
        r.set_option("sample_budget", 0)
    # sampling_view still draws the sampling net's view
    r.set_option("sampling_view", 1)
    try:
        v = r.render_rays(pose, torch.eye(3), dirs, 0.5, 8, want_oracle_weights=True)
        assert torch.equal(v["rgb"], r.sampling_view(v["oracle_weights"], rgba8=False)["rgb"])
    finally:
        r.set_option("sampling_view", 0)


def test_adaptive_path_unchanged_on_the_same_context(pav):
    r, scene, _, _ = pav
    dirs = r.generate_ray_directions(200, 150)
    pose = torch.tensor(scene["view_cell_center"])
    r.set_option("sampler", 0)
    a = r.render_rays(pose, torch.eye(3), dirs, 0.15, 16, want_aux=True)
    r.set_option("sampler", 1)
    d = r.render_rays(pose, torch.eye(3), dirs, 0.15, 16)
    r.set_option("sampler", 0)
    b = r.render_rays(pose, torch.eye(3), dirs, 0.15, 16, want_aux=True)
    r.set_option("sampler", 1)
    for k in ("rgb", "n_samples") + r.AUX_KEYS:
        assert _same(a[k], b[k]), k
    assert not torch.equal(a["rgb"], d["rgb"])


def test_export_dir_and_adapter(tmp_path):
    """convert's DONeRF export through Renderer.from_export_dir, and the TrainConfig.inference drop-in's dict keys."""
    from adanerf_b200 import Renderer
    from adanerf_b200.adapter import B200Inference
    sd0, sd1 = orc.make_weights("rand", seed=100)
    d = tmp_path / "export"
    ow.write_export_dir(str(d), orc.SCENE_BARBERSHOP, sd0, sd1, 0.0, 8, sampler="FromClassifiedDepth",
                        sampling_loss="CrossEntropyLoss")
    r, thr, K = Renderer.from_export_dir(str(d))
    ref, _, _, _ = _renderer("rand", transform=2)
    dirs = r.generate_ray_directions(64, 48)
    pose = torch.tensor(orc.SCENE_BARBERSHOP["view_cell_center"])
    a = r.render_rays(pose, torch.eye(3), dirs, thr, K)
    b = ref.render_rays(pose, torch.eye(3), dirs, thr, K)
    assert K == 8 and torch.equal(a["rgb"], b["rgb"])
    inf = B200Inference(orc.SCENE_BARBERSHOP, sd0, sd1, 0.0, 8, sampler=1, pdf_transform=2)
    batch = {"ImagePose": pose[None], "ImageRotation": torch.eye(3)[None], "RayDirectionsSamples": dirs[None]}
    outs, dicts = inf.inference(batch)
    assert torch.equal(outs[1], b["rgb"])
    assert "AdaptiveSamplePositions" not in dicts[1] and "OracleWeights" not in dicts[1]
    r.close()
    ref.close()


def test_headless_viewer_renders_donerf_export(tmp_path):
    import __graft_entry__ as g
    sd0, sd1 = load_weights_npz(os.path.join(GOLDEN, "weights_pavillon"))
    d = tmp_path / "export"
    ow.write_export_dir(str(d), orc.SCENE_PAVILLON, sd0, sd1, 0.0, 8, sampler="FromClassifiedDepth")
    for extra in ([], ["--surface"]):
        res = subprocess.run([g.VIEWER, str(d), "-s", "400", "300", "-f", "3", "-w"] + extra, capture_output=True, text=True,
                             timeout=300)
        assert res.returncode == 0, res.stderr
        m = re.search(r"frames 400x300: ([0-9.]+) ms/frame .*\(([0-9.]+) per ray", res.stdout)
        assert m and abs(float(m.group(2)) - 8.0) < 1e-6, res.stdout


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_multi_gpu_bands_equal_single_frame(pav):
    from adanerf_b200.multi import MultiRenderer
    r, scene, sd0, sd1 = pav
    W, H, K = 320, 241, 8
    pose = torch.tensor(scene["view_cell_center"])
    single = r.render_camera(pose, torch.eye(3), W, H, 0.5, K)["rgb"]
    m = MultiRenderer(scene, [0, 1], sd0, sd1)
    m.set_option("sampler", 1)
    m.set_option("pdf_transform", 1)
    m.render_camera(pose, torch.eye(3), W, H, 0.5, K)
    assert torch.equal(m.wait_frame().clone(), single)
    m.close()
