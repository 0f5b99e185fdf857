"""Networks trained with D = 32, 64 or 256 depth cells (multiDepthFeatures) on the H100.

  * stage 2 (stage2_cells_kernel) and the sample-budget select (budget_keys_cells_kernel) bit for bit against the CPU
    restatement, on whole 800x800 frames of a D-output sampling net at every K edge, with ties and a partial last tile,
    and across launches alternating D on two contexts;
  * the surface entry, row bands on one device and a budget group of one at D != 128;
  * a budgeted render equals the render at the threshold it reports;
  * every render entry, views call and *_host entry equals the stage entries composed by hand (dense mode at K = D = 64
    included);
  * end to end against the reference's fixtures (oracle/gen_cells_golden.py);
  * the refusals, and a D = 256 export directory through adn_create_from_export_dir and the headless viewer."""
import os
import subprocess

import numpy as np
import pytest
import torch

from conftest import ROOT, load_golden
from oracle import adanerf_oracle as orc
from oracle import cells_oracle as co
from oracle import stage_emulation as se
from oracle.gen_cells_golden import CASES, case_inputs
from test_sample_budget_oracle import budget_threshold
from test_selection_exact import _with_extreme_rows, check_stage2

pytestmark = pytest.mark.gpu

F32 = np.float32
W = H = 800
# the K at which the kernels' paths switch or end, per D
K_EDGES = {32: [1, 2, 16, 31, 32], 64: [1, 8, 33, 63, 64], 256: [1, 16, 17, 100, 128]}


def _renderer(scene, sd0=None, sd1=None):
    from adanerf_b200 import Renderer
    return Renderer(scene, device=0, sampling_net=sd0, shading_net=sd1)


def _bits(a):
    return np.ascontiguousarray(np.asarray(a, F32)).view(np.uint32)


def _frame_raw0(D, seed=0):
    """raw0 [640000, D] of a shaped D-output net over a whole frame, with rows moved above / below every threshold."""
    scene = orc.SCENE_BARBERSHOP
    sd0, _ = co.make_weights(D, "shaped", seed=seed)
    r = _renderer(scene, sd0)
    pose = np.asarray(scene["view_cell_center"], F32) + np.asarray((0.1, -0.05, 0.02), F32)
    x0, _, _ = r.stage0(pose, orc.rotation_yaw(30.0), r.generate_ray_directions(W, H))
    raw0 = r.mlp0(x0)
    assert raw0.shape == (W * H, D) and r.depth_cells() == D and r.net_dims(0) == (90, D)
    out = _with_extreme_rows(raw0.cpu())
    return r, out


@pytest.fixture(scope="module")
def frames():
    return {D: _frame_raw0(D) for D in (32, 64, 256)}


def _thresholds(raw0, K):
    srt = torch.sort(raw0[::7], dim=1, descending=True).values
    out = []
    for j in (K, max(K // 2, 1)):
        t = F32(torch.median(srt[:, j - 1]).item())
        out.append(float(t) if t > 0 else 2.0 ** -6)
    return out


@pytest.mark.parametrize("D", [32, 64, 256])
def test_stage2_whole_frame_bit_exact(frames, D):
    r, raw0 = frames[D]
    lut = co.zlut(orc.SCENE_BARBERSHOP, D)
    dev = raw0.cuda()
    for K in K_EDGES[D]:
        for thr in _thresholds(raw0, K):
            check_stage2(r, dev, raw0, thr, K, lut, f"D={D} K={K} thr={thr}")


@pytest.mark.parametrize("D", [32, 64, 256])
def test_stage2_ties_and_partial_tile(frames, D):
    """raw0 rounded to multiples of 1/16 (exact ties everywhere), 37 extra rows: N = 640 037, a partial last tile."""
    r, raw0 = frames[D]
    v = torch.round(torch.cat([raw0, raw0[:37] * 0.5]) * 16) / 16
    lut = co.zlut(orc.SCENE_BARBERSHOP, D)
    dev = v.cuda()
    for K in (1, min(D, 128) // 4, min(D, 128)):
        check_stage2(r, dev, v, 0.25, K, lut, f"ties D={D} K={K}")
    # a 4-byte aligned view gives the same result (the cells kernels load 4-byte words)
    shifted = torch.empty(v.numel() + 1, device="cuda")[1:].view(v.shape)
    shifted.copy_(dev)
    a, b = r.stage2(dev, 0.25, 8), r.stage2(shifted, 0.25, 8)
    for k in ("count", "offset", "cell", "ray", "z", "zp"):
        assert torch.equal(a[k], b[k]), k


@pytest.mark.parametrize("D", [32, 64, 256])
def test_budget_threshold_bit_exact(frames, D):
    r, raw0 = frames[D]
    raw0 = raw0[:200_003]
    dev = raw0.cuda()
    for K in K_EDGES[D][1:]:
        n = raw0.shape[0]
        for B in (n, n + n * (K - 1) // 10, n + n * (K - 1) // 2, n * K + 5):
            got = r.budget_threshold(dev, 0.1, K, B).item()
            assert _bits(got) == _bits(budget_threshold(raw0, 0.1, K, B)), (D, K, B)


def test_launch_sequences_across_D_on_two_contexts(frames):
    """Stage 2 and the budget alternating between a D = 32 and a D = 256 context give what each call gives on its own."""
    (ra, a), (rb, b) = frames[32], frames[256]
    a, b = a[:100_000].cuda(), b[:77_777].cuda()
    want = {"a": ra.stage2(a, 0.2, 8), "b": rb.stage2(b, 0.2, 100)}
    ta = ra.budget_threshold(a, 0.2, 32, 500_000).item()
    tb = rb.budget_threshold(b, 0.2, 16, 200_000).item()
    for _ in range(3):
        got_a = ra.stage2(a, 0.2, 8)
        assert rb.budget_threshold(b, 0.2, 16, 200_000).item() == tb
        got_b = rb.stage2(b, 0.2, 100)
        assert ra.budget_threshold(a, 0.2, 32, 500_000).item() == ta
        for k in ("count", "offset", "cell", "ray", "z", "zp"):
            assert torch.equal(got_a[k], want["a"][k]) and torch.equal(got_b[k], want["b"][k]), k


# ------------------------------------------------------------------------------------------------ render entries
def _net_renderer(D, scene=orc.SCENE_PAVILLON, kind="shaped", seed=1):
    sd0, sd1 = co.make_weights(D, kind, seed=seed)
    return _renderer(scene, sd0, sd1), sd0, sd1


def _same(a, b):
    """Equal bits (NaN padding included)."""
    if a.dtype == torch.float32:
        return a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))
    return torch.equal(a, b)


def _compose(r, scene, pose, rot, dirs, thr, K):
    """A frame from the stage entries: stage 0 -> mlp0 -> stage 2 (or dense) -> stage 3 -> mlp1 -> stage 5."""
    x0, ro, rd = r.stage0(pose, rot, dirs)
    raw0 = r.mlp0(x0)
    n = raw0.shape[0]
    if thr == 0.0:
        lut = torch.from_numpy(se.zlut_dense(scene, K)).cuda()
        ray = torch.arange(n, device="cuda", dtype=torch.int32).repeat_interleave(K)
        x1 = r.stage3(ro, rd, ray, lut.repeat(n))
        out = r.stage5(r.mlp1(x1), raw0, None, None, None, K, dense=True, aux=True, rgba8=True)
        out["n_samples"] = torch.full((n,), K, dtype=torch.int32, device="cuda")
    else:
        s2 = r.stage2(raw0, thr, K)
        x1 = r.stage3(ro, rd, s2["ray"], s2["z"])
        out = r.stage5(r.mlp1(x1), s2["zp"], s2["z"], s2["offset"], s2["count"], K, aux=True, rgba8=True)
        out["n_samples"] = s2["count"]
    out["raw0"] = raw0
    return out


@pytest.mark.parametrize("D,K,thr", [(32, 8, 0.2), (32, 32, 0.2), (64, 16, 0.2), (64, 64, 0.0), (256, 16, 0.2), (256, 128, 0.2)])
def test_every_entry_equals_the_stages(D, K, thr):
    scene = orc.SCENE_PAVILLON
    r, _, _ = _net_renderer(D, scene)
    Wc, Hc = 96, 64
    pose = torch.tensor(scene["view_cell_center"]) + torch.tensor([0.03, -0.02, 0.01])
    rot = orc.rotation_yaw(40.0)
    dirs = r.generate_ray_directions(Wc, Hc)
    want = _compose(r, scene, pose, rot, dirs, thr, K)
    n = dirs.shape[0]
    got = r.render_rays(pose, rot, dirs, thr, K, want_oracle_weights=True, want_aux=True)
    assert got["oracle_weights"].shape == (n, D)
    assert torch.equal(got["oracle_weights"], want["raw0"])
    for k in ("rgb", "n_samples") + r.AUX_KEYS:
        assert _same(got[k], want[k]), k
    r.set_option("chunk_rays", 1024)   # several chunks: raw0 rows and outputs at every chunk offset
    got = r.render_rays(pose, rot, dirs, thr, K, want_oracle_weights=True, want_aux=("weights", "depth_map"))
    assert torch.equal(got["oracle_weights"], want["raw0"]) and torch.equal(got["rgb"], want["rgb"])
    assert _same(got["weights"], want["weights"]) and _same(got["depth_map"], want["depth_map"])
    r.set_option("chunk_rays", 0)
    cam = r.render_camera(pose, rot, Wc, Hc, thr, K, want_nsamples=True)
    assert torch.equal(cam["rgb"], want["rgb"]) and torch.equal(cam["n_samples"], want["n_samples"])
    assert torch.equal(r.render_camera_rgba8(pose, rot, Wc, Hc, thr, K), want["rgba8"])
    host = r.render_rays_host(pose, rot, dirs.cpu().numpy(), thr, K)
    np.testing.assert_array_equal(host["rgb"], want["rgb"].cpu().numpy())
    host = r.render_camera_host(pose, rot, Wc, Hc, thr, K, want_nsamples=True)
    np.testing.assert_array_equal(host["rgb"], want["rgb"].cpu().numpy())
    # two views in one call: the single-view calls concatenated
    pose2, rot2 = pose + torch.tensor([-0.05, 0.04, 0.0]), orc.rotation_yaw(-70.0)
    want2 = _compose(r, scene, pose2, rot2, dirs, thr, K)
    v = r.render_views(torch.stack([pose, pose2]), torch.stack([rot, rot2]), torch.stack([dirs, dirs]), thr, K,
                       want_oracle_weights=True)
    assert torch.equal(v["rgb"], torch.cat([want["rgb"], want2["rgb"]]))
    assert torch.equal(v["oracle_weights"], torch.cat([want["raw0"], want2["raw0"]]))
    vc = r.render_views_camera(torch.stack([pose, pose2]), torch.stack([rot, rot2]), Wc, Hc, thr, K)
    assert torch.equal(vc["rgb"], torch.cat([want["rgb"], want2["rgb"]]))
    r.close()


@pytest.mark.parametrize("D,K", [(32, 16), (64, 48), (256, 100)])
def test_budgeted_render_is_the_render_at_its_threshold(D, K):
    r, _, _ = _net_renderer(D, orc.SCENE_BARBERSHOP)
    pose, rot = torch.tensor(orc.SCENE_BARBERSHOP["view_cell_center"]), orc.rotation_yaw(10.0)
    Wc, Hc = 200, 120
    free = r.render_camera(pose, rot, Wc, Hc, 0.1, K, want_nsamples=True)
    B = Wc * Hc + int(free["n_samples"].sum().item() - Wc * Hc) // 3
    r.set_option("sample_budget", B)
    r.set_option("chunk_rays", 8192)
    got = r.render_camera(pose, rot, Wc, Hc, 0.1, K, want_nsamples=True)
    t = r.last_threshold()
    assert int(got["n_samples"].sum()) <= B and t > 0.1
    r.set_option("sample_budget", 0)
    r.set_option("chunk_rays", 0)
    at = r.render_camera(pose, rot, Wc, Hc, t, K, want_nsamples=True)
    assert torch.equal(got["rgb"], at["rgb"]) and torch.equal(got["n_samples"], at["n_samples"])
    r.close()


@pytest.mark.parametrize("D", [32, 256])
def test_surface_row_bands_and_budget_group(D):
    """The paths that reach render() from elsewhere, at D != 128: the surface entry writes the rgba8 entry's pixels; the
    row-band renderer on one device gives the single-context frame; a budgeted call as the only member of a budget group
    (a reducer that leaves the words as they are) renders the ungrouped budgeted frame at the same threshold."""
    from adanerf_b200.multi import MultiRenderer
    from adanerf_b200.renderer import _fptr
    from test_stream_order import Surface
    scene = orc.SCENE_BARBERSHOP
    r, sd0, sd1 = _net_renderer(D, scene)
    pose, rot = torch.tensor(scene["view_cell_center"]), orc.rotation_yaw(25.0)
    Wc, Hc, K = 160, 100, 16
    px = r.render_camera_rgba8(pose, rot, Wc, Hc, 0.2, K)
    surf = Surface(Wc, Hc)
    p, q = r._pose_rot(pose, rot)
    r._check(r.lib.adn_render_camera_surface(r.handle, _fptr(p), _fptr(q), Wc, Hc, 0, Hc, 0.2, K, surf.surf.value, r._stream()))
    torch.cuda.synchronize()
    assert np.array_equal(surf.read().reshape(-1, 4), px.cpu().numpy())
    surf.free()
    want = r.render_camera(pose, rot, Wc, Hc, 0.2, K)["rgb"].cpu()
    m = MultiRenderer(scene, [0], sd0, sd1)
    m.render_camera(pose, rot, Wc, Hc, 0.2, K)
    assert torch.equal(m.wait_frame().cpu(), want)
    m.close()
    free = r.render_camera(pose, rot, Wc, Hc, 0.1, K, want_nsamples=True)
    B = Wc * Hc + int(free["n_samples"].sum().item() - Wc * Hc) // 3
    r.set_option("sample_budget", B)
    alone = r.render_camera(pose, rot, Wc, Hc, 0.1, K, want_nsamples=True)
    t_alone = r.last_threshold()
    r.set_budget_group(lambda words: None)
    grouped = r.render_camera(pose, rot, Wc, Hc, 0.1, K, want_nsamples=True)
    assert r.last_threshold() == t_alone > 0.1 and int(grouped["n_samples"].sum()) <= B
    assert torch.equal(grouped["rgb"], alone["rgb"]) and torch.equal(grouped["n_samples"], alone["n_samples"])
    r.set_budget_group(None)
    r.close()


# ------------------------------------------------------------------------------------------------ against the fixtures
@pytest.mark.parametrize("name", list(CASES))
def test_end_to_end_against_reference_fixtures(name):
    """One render against the reference's colours: |dPSNR| < 0.05 dB against a common image (the reference's colours plus
    fixed noise of sigma 0.03, a ~30 dB image; the bar of tests/test_views_gpu.py), PSNR >= 49.4 dB against the reference
    over all rays (tests/test_parity_gate.py), and, for the adaptive sampler, the reference's sample count on >= 99.9 % of
    the rays; on the rays whose sample count agrees every colour channel is within 5e-3 of the reference's (bf16 shading
    MLP; 7.1e-4 at most measured on an H100)."""
    g = load_golden(f"cells_{name}")
    m = g["meta"]
    scene, pose, rot, dirs, sd0, sd1 = case_inputs(name, m["case"]["seed"])
    r = _renderer(scene, sd0, sd1)
    out = r.render_rays(pose, rot, dirs.cuda(), m["thr"], m["K"], want_oracle_weights=True)
    np.testing.assert_allclose(out["oracle_weights"].cpu().numpy(), g["raw0"], rtol=0, atol=2e-3)
    rgb = out["rgb"].cpu().numpy()
    same = np.ones(rgb.shape[0], bool)
    if m["thr"] > 0:
        same = (out["n_samples"].cpu().numpy() / m["K"]).astype(F32) == g["asp"]
        assert same.mean() >= 0.999
    psnr = lambda a, b: 10.0 * np.log10(1.0 / np.mean((np.asarray(a, np.float64) - np.asarray(b, np.float64)) ** 2))
    common = g["rgb"] + np.random.default_rng(0).normal(0.0, 0.03, g["rgb"].shape)
    d_psnr = psnr(rgb, common) - psnr(g["rgb"], common)
    worst = float(np.abs(rgb - g["rgb"])[same].max())
    print(f"{name}: dPSNR {d_psnr:+.5f} dB, PSNR vs the reference {psnr(rgb, g['rgb']):.2f} dB, "
          f"same sample count {same.mean():.4f}, max |d rgb| on those rays {worst:.2e}")
    assert abs(d_psnr) < 0.05
    assert psnr(rgb, g["rgb"]) >= 49.4
    assert worst < 5e-3
    r.close()


# ------------------------------------------------------------------------------------------------ refusals
def test_refusals():
    from adanerf_b200 import AdnError
    r, _, _ = _net_renderer(64)
    pose, rot = torch.tensor(orc.SCENE_PAVILLON["view_cell_center"]), torch.eye(3)
    dirs = r.generate_ray_directions(16, 16)
    with pytest.raises(AdnError, match="K <= 64") as e:
        r.render_rays(pose, rot, dirs, 0.2, 65)
    assert e.value.status == 1
    with pytest.raises(AdnError, match="K == 64") as e:
        r.render_rays(pose, rot, dirs, 0.0, 32)                   # dense mode needs K = D
    assert e.value.status == 1
    r.set_option("sampler", 1)
    with pytest.raises(AdnError, match="sampler 1") as e:
        r.render_rays(pose, rot, dirs, 0.0, 8)
    assert e.value.status == 1
    r.set_option("sampler", 0)
    r.set_option("sampling_view", 1)
    with pytest.raises(AdnError, match="sampling_view") as e:
        r.render_rays(pose, rot, dirs, 0.2, 8)
    assert e.value.status == 1
    r.set_option("sampling_view", 0)
    with pytest.raises(AdnError, match="K <= 64"):
        r.stage2(torch.zeros(4, 64, device="cuda"), 0.2, 65)
    with pytest.raises(ValueError, match="64"):
        r.stage2(torch.zeros(4, 128, device="cuda"), 0.2, 8)
    r.close()
    r, _, _ = _net_renderer(256)
    with pytest.raises(AdnError, match="256 depth cells have no dense mode") as e:
        r.render_rays(pose, rot, dirs, 0.0, 128)
    assert e.value.status == 1
    r.close()
    with pytest.raises(AdnError, match="32, 64, 128 or 256"):
        _net_renderer(48)


def test_export_dir_with_256_cells_renders_and_views(tmp_path):
    from adanerf_b200 import Renderer
    from adanerf_b200 import onnx_weights as ow
    scene = orc.SCENE_PAVILLON
    sd0, sd1 = co.make_weights(256, "shaped", seed=2)
    d = tmp_path / "d256"
    ow.write_export_dir(str(d), scene, sd0, sd1, 0.2, 16)
    r, thr, K = Renderer.from_export_dir(str(d))
    assert r.depth_cells() == 256 and (thr, K) == (pytest.approx(0.2), 16)
    direct = _renderer(scene, sd0, sd1)
    pose, rot = torch.tensor(scene["view_cell_center"]), orc.rotation_yaw(15.0)
    a = r.render_camera(pose, rot, 64, 48, thr, K)["rgb"]
    b = direct.render_camera(pose, rot, 64, 48, thr, K)["rgb"]
    assert torch.equal(a, b)
    r.close()
    direct.close()
    viewer = os.path.join(ROOT, "adanerf_b200", "adn_viewer_headless")
    p = subprocess.run([viewer, str(d), "-s", "96", "64", "-f", "2"], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stdout + p.stderr
    assert "net 0: sampling 8 x 256, skip -1, posEnc 10-4, 256 depth cells" in p.stdout, p.stdout
    # a config whose multiDepthFeatures disagrees with model0.onnx is refused when the networks are built
    cfg = (d / "config.ini").read_text().replace("multiDepthFeatures = [256, 256]", "multiDepthFeatures = [64, 64]")
    (d / "config.ini").write_text(cfg)
    from adanerf_b200 import AdnError
    with pytest.raises(AdnError) as e:
        Renderer.from_export_dir(str(d))
    assert e.value.status == 5
