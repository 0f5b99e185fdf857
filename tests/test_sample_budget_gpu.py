"""Sample budget on the GPU (adn_set_option "sample_budget", adn_budget_threshold, adn_last_threshold): the threshold chosen
on the device equals the oracle's bit for bit, and a budgeted render is bit-identical to a fixed-threshold render at that
threshold, on one chunk and across chunks, through the rays / camera / rgba8 / host entry points."""
import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import adanerf_oracle as orc
from test_sample_budget_oracle import KS, SETS, budget_threshold, budgets

pytestmark = pytest.mark.gpu


def _renderer(scene, sd0=None, sd1=None):
    from adanerf_b200 import Renderer
    return Renderer(scene, device=0, sampling_net=sd0, shading_net=sd1)


def _bits(t):
    return np.float32(t).view(np.uint32)


@pytest.fixture(scope="module")
def bare():
    r = _renderer(orc.SCENE_BARBERSHOP)
    yield r
    r.close()


@pytest.fixture(scope="module")
def pav(pavillon_weights):
    sd0, sd1 = pavillon_weights
    r = _renderer(orc.SCENE_PAVILLON, sd0, sd1)
    yield r
    r.close()


def _pav_view():
    pose = torch.tensor(orc.SCENE_PAVILLON["view_cell_center"]) + torch.tensor([0.05, -0.03, 0.02])
    rot = torch.tensor([[1, 0, 0], [0, 0, -1], [0, 1, 0]], dtype=torch.float32)
    return pose, rot


@pytest.mark.parametrize("K", KS)
@pytest.mark.parametrize("name", sorted(SETS))
def test_device_threshold_equals_oracle_on_golden_raw0(bare, name, K):
    raw0 = torch.from_numpy(load_golden(name)["raw0"])
    thr_min = SETS[name]
    for label, B in budgets(raw0, thr_min, K).items():
        got = bare.budget_threshold(raw0.cuda(), thr_min, K, B).item()
        want = budget_threshold(raw0, thr_min, K, B)
        assert _bits(got) == _bits(want), (label, B, got, float(want))


@pytest.mark.parametrize("K", [8, 16, 32])
def test_device_threshold_equals_oracle_at_frame_size(bare, K):
    """Many CTAs flushing into the histograms (K = 32: the warp-per-ray extraction)."""
    g = torch.Generator().manual_seed(K)
    n = 200_000
    raw0 = torch.rand(n, 128, generator=g) * 1.5 - 0.5
    for B in (n + (n * (K - 1)) // 3, 3 * n):
        want = budget_threshold(raw0, 0.2, K, B)
        assert _bits(bare.budget_threshold(raw0.cuda(), 0.2, K, B).item()) == _bits(want), B


def test_budget_render_one_chunk_equals_fixed_threshold(pav):
    """K = 8, 20 000 rays (one chunk): budgeted render == fixed-threshold render at t*, also with the auxiliary outputs and
    through the host-buffer entry; t* is the oracle's on the raw0 of the call."""
    pose, rot = _pav_view()
    dirs = torch.from_numpy(orc.generate_ray_directions(800, 800, orc.SCENE_PAVILLON["fov"]).reshape(-1, 3)).float()[::31][:20000]
    n, K, thr_min = dirs.shape[0], 8, 0.05
    B = 4 * n
    pav.set_option("sample_budget", B)
    out = pav.render_rays(pose, rot, dirs.cuda(), thr_min, K, want_oracle_weights=True)
    t = pav.last_threshold()
    aux = pav.render_rays(pose, rot, dirs.cuda(), thr_min, K, want_aux=True)
    host = pav.render_rays_host(pose, rot, dirs.numpy(), thr_min, K)
    pav.set_option("sample_budget", 0)
    fixed = pav.render_rays(pose, rot, dirs.cuda(), t, K)
    assert _bits(t) == _bits(budget_threshold(out["oracle_weights"].cpu(), thr_min, K, B))
    assert t > thr_min                                       # the budget binds: the floor saturates every ray at K
    m = int(out["n_samples"].long().sum())
    print(f"one chunk: t* = {t:.6f}, M = {m} <= B = {B}")
    assert m <= B
    assert torch.equal(out["rgb"], fixed["rgb"]) and torch.equal(out["n_samples"], fixed["n_samples"])
    assert torch.equal(aux["rgb"], fixed["rgb"])
    np.testing.assert_array_equal(host["rgb"], fixed["rgb"].cpu().numpy())
    np.testing.assert_array_equal(host["n_samples"], fixed["n_samples"].cpu().numpy())


def test_budget_render_full_frame_two_chunks(pav):
    """K = 16 on an 800x800 camera frame: two internal chunks share one threshold.  Camera, rays (raw0 in the caller's
    d_oracle_weights) and rgba8 entries agree with each other and with the fixed-threshold frame at t*."""
    pose, rot = _pav_view()
    W = H = 800
    K, thr_min = 16, 0.05
    n = W * H
    B = 8 * n
    pav.set_option("sample_budget", B)
    cam = pav.render_camera(pose, rot, W, H, thr_min, K, want_nsamples=True)
    t_cam = pav.last_threshold()
    rays = pav.render_rays(pose, rot, pav.generate_ray_directions(W, H), thr_min, K, want_oracle_weights=True)
    t_rays = pav.last_threshold()
    rgba = pav.render_camera_rgba8(pose, rot, W, H, thr_min, K)
    pav.set_option("sample_budget", 0)
    fixed = pav.render_camera(pose, rot, W, H, t_cam, K, want_nsamples=True)
    fixed_rgba = pav.render_camera_rgba8(pose, rot, W, H, t_cam, K)
    m = int(cam["n_samples"].long().sum())
    print(f"800x800 K=16: t* = {t_cam:.6f}, M = {m} <= B = {B}")
    assert _bits(t_cam) == _bits(t_rays)
    assert _bits(t_rays) == _bits(budget_threshold(rays["oracle_weights"].cpu(), thr_min, K, B))
    assert thr_min < t_cam and m <= B
    assert torch.equal(cam["rgb"], fixed["rgb"]) and torch.equal(cam["n_samples"], fixed["n_samples"])
    assert torch.equal(rays["rgb"], fixed["rgb"]) and torch.equal(rays["n_samples"], fixed["n_samples"])
    assert torch.equal(rgba, fixed_rgba)


def test_budget_that_never_binds_is_the_fixed_frame(pav):
    pose, rot = _pav_view()
    W, H, K, thr = 800, 200, 8, 0.3
    plain = pav.render_camera(pose, rot, W, H, thr, K, want_nsamples=True)
    pav.set_option("sample_budget", W * H * K)
    loose = pav.render_camera(pose, rot, W, H, thr, K, want_nsamples=True)
    t = pav.last_threshold()
    pav.set_option("sample_budget", 0)
    assert _bits(t) == _bits(thr)
    assert torch.equal(plain["rgb"], loose["rgb"]) and torch.equal(plain["n_samples"], loose["n_samples"])


def test_budget_error_paths_and_switching_off(pav):
    from adanerf_b200 import AdnError
    pose, rot = _pav_view()
    W, H = 64, 32
    base = pav.render_camera(pose, rot, W, H, 0.2, 8)
    pav.set_option("sample_budget", W * H - 1)              # B < N
    with pytest.raises(AdnError, match="below") as e:
        pav.render_camera(pose, rot, W, H, 0.2, 8)
    assert e.value.status == 1
    pav.set_option("sample_budget", W * H * 128)
    with pytest.raises(AdnError, match="dense") as e:       # thr == 0: dense mode has no threshold to choose
        pav.render_camera(pose, rot, W, H, 0.0, 128)
    assert e.value.status == 1
    with pytest.raises(AdnError):
        pav.set_option("sample_budget", -1)
    with pytest.raises(AdnError):
        pav.budget_threshold(torch.zeros(4, 128, device="cuda"), 0.2, 8, 3)
    flat = torch.zeros(4 * 128 + 1, device="cuda")
    with pytest.raises(AdnError, match="aligned") as e:    # rows are read as 16-byte vectors, like stage 2 reads them
        pav.budget_threshold(flat[1:].view(4, 128), 0.2, 8, 8)
    assert e.value.status == 1
    pav.set_option("sample_budget", 0)
    again = pav.render_camera(pose, rot, W, H, 0.2, 8)
    assert torch.equal(base["rgb"], again["rgb"]) and pav.last_threshold() == np.float32(0.2)


def test_budget_selection_is_timed_with_stage2(pav):
    pose, rot = _pav_view()
    pav.set_option("profile", 1)
    pav.set_option("sample_budget", 4 * 800 * 100)
    pav.render_camera(pose, rot, 800, 100, 0.05, 8)
    st = pav.stats()
    pav.set_option("sample_budget", 0)
    pav.set_option("profile", 0)
    assert all(ms > 0 for ms in st["ms_stage"]), st["ms_stage"]


def test_viewer_budget_prints_threshold_and_samples(tmp_path):
    """adn_viewer_headless --budget SAMPLES_PER_FRAME: every timed frame reports its threshold and M <= the budget."""
    import re
    import subprocess
    import __graft_entry__ as g
    from adanerf_b200 import onnx_weights as ow
    g.build()
    sd0, sd1 = orc.make_weights("shaped", seed=0)
    d = tmp_path / "export"
    ow.write_export_dir(str(d), orc.SCENE_BARBERSHOP, sd0, sd1, 0.2, 8)
    budget = 400 * 300 * 3
    r = subprocess.run([g.VIEWER, str(d), "-s", "400", "300", "-f", "3", "--budget", str(budget)], capture_output=True, text=True,
                       timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    frames = re.findall(r"frame \d+: threshold ([0-9.e+-]+), (\d+) samples \(budget (\d+)\)", r.stdout)
    assert len(frames) == 3, r.stdout
    for thr, m, b in frames:
        assert float(thr) >= np.float32(0.2) and int(m) <= int(b) == budget
