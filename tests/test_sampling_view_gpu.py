"""The sampling network's view on the H100 (option "sampling_view", adn_sampling_view): the kernel against the reference
viewer's own samplesToImage (oracle/_ref/libref_viewer_kernels.so, built by oracle/ref_viewer.py) and the numpy emulation
(oracle/sampling_view.py) byte for byte; full frames of the two shipped exports through every render entry; the option
leaving normal renders alone; call order; the headless viewer's --oracle."""
import ctypes as C
import json
import os
import subprocess
import threading
import time

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import adanerf_oracle as orc
from oracle import ref_viewer
from oracle import sampling_view as sv
from test_sampling_view import crafted_rows

pytestmark = pytest.mark.gpu

W = H = 800
RX = torch.tensor([[1, 0, 0], [0, 0, -1], [0, 1, 0]], dtype=torch.float32)   # camera -z -> world +y
POSES = {"barbershop_k4": ([0.3, -0.2, 0.08], 35.0), "pavillon_k16": ([0.05, -0.03, 0.02], 0.0)}
ADN_ERR_INVALID = 1


def _bytes(t):
    a = t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)
    return np.ascontiguousarray(a).view(np.uint8)


def _same(a, b, what):
    a, b = _bytes(a), _bytes(b)
    assert a.shape == b.shape, (what, a.shape, b.shape)
    n = int((a != b).sum())
    assert n == 0, f"{what}: {n} bytes differ"


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as g
    g.build()
    return g


@pytest.fixture(scope="module")
def exports(tmp_path_factory):
    """name -> the shipped export directory reassembled from its parts under tests/golden/shipped/."""
    out = {}
    for name in POSES:
        src = os.path.join(GOLDEN, "shipped", name)
        with open(os.path.join(src, "manifest.json")) as f:
            man = json.load(f)
        dst = tmp_path_factory.mktemp(name)
        for fname, e in man["files"].items():
            data = b""
            for p in e.get("parts", [fname]):
                with open(os.path.join(src, p), "rb") as f:
                    data += f.read()
            (dst / fname).write_bytes(data)
        out[name] = str(dst)
    return out


def _pose_rot(name):
    from oracle.adanerf_oracle import SCENE_BARBERSHOP, SCENE_PAVILLON
    scene = SCENE_BARBERSHOP if name.startswith("barber") else SCENE_PAVILLON
    off, yaw = POSES[name]
    return torch.tensor(scene["view_cell_center"]) + torch.tensor(off), orc.rotation_yaw(yaw) @ RX


def _crafted(n, seed=0):
    rows = crafted_rows(seed)
    if n <= len(rows):
        return rows[:n].copy()
    rng = np.random.default_rng(seed + 1)
    rest = rng.standard_normal((n - len(rows), 128)).astype(np.float32)
    rest[::7] = np.round(rest[::7])                                   # many ties
    pick = rng.integers(0, len(rows), n // 16)
    rest[rng.integers(0, len(rest), len(pick))] = rows[pick]         # crafted rows scattered through the frame
    return np.concatenate([rows, rest])


# ---- the kernel against the reference viewer's ----------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ref_lib(built):
    if not os.path.exists(ref_viewer.LIB):
        pytest.skip(f"{ref_viewer.LIB} is absent: build() makes it only where a reference checkout exists")
    lib = C.CDLL(ref_viewer.LIB)
    lib.ref_sampling_view.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    return lib


@pytest.fixture(scope="module")
def renderer(built):
    from adanerf_b200 import Renderer
    sd0, sd1 = orc.make_weights("shaped", seed=0)
    r = Renderer(orc.SCENE_BARBERSHOP, device=0, sampling_net=sd0, shading_net=sd1)
    yield r
    r.close()


@pytest.mark.parametrize("n", [1, 127, 128, 129, 640_000])
def test_stage_entry_equals_reference_kernel_and_emulation(ref_lib, renderer, n):
    raw0 = _crafted(n)
    d_raw0 = torch.from_numpy(raw0).cuda()
    width = min(n, W)
    ref_px = torch.full((n, 4), 7, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    assert ref_lib.ref_sampling_view(d_raw0.data_ptr(), n, width, ref_px.data_ptr()) == 0
    out = renderer.sampling_view(d_raw0)
    torch.cuda.synchronize()
    rgb, px = sv.sampling_view(raw0)
    _same(out["rgba8"], ref_px, "pixels vs the reference kernel")
    _same(out["rgba8"], px, "pixels vs the emulation")
    _same(out["rgb"], rgb, "fp32 view vs the emulation")
    one = renderer.sampling_view(d_raw0, rgb=False)                  # either output alone
    assert one["rgb"] is None
    _same(one["rgba8"], px, "pixels alone")


def test_stage_entry_refuses_bad_arguments(renderer):
    from adanerf_b200 import AdnError
    raw0 = torch.zeros((65, 128), device="cuda")
    for args in ((raw0.data_ptr() + 4, 64, raw0.data_ptr(), None),   # unaligned rows
                 (raw0.data_ptr(), 64, None, None),                   # no output
                 (None, 64, raw0.data_ptr(), None)):                  # no input
        with pytest.raises(AdnError) as e:
            renderer._check(renderer.lib.adn_sampling_view(renderer.handle, *args))
        assert e.value.status == ADN_ERR_INVALID


# ---- full frames of the shipped exports --------------------------------------------------------------------------------------
@pytest.fixture(scope="module", params=sorted(POSES))
def shipped(request, built, exports):
    from adanerf_b200 import Renderer
    name = request.param
    r, thr, K = Renderer.from_export_dir(exports[name])
    r.set_option("sampling_view", 1)
    pose, rot = _pose_rot(name)
    dirs = r.generate_ray_directions(W, H)
    o = r.render_rays(pose, rot, dirs, thr, K, want_oracle_weights=True)
    torch.cuda.synchronize()
    yield dict(r=r, thr=thr, K=K, pose=pose, rot=rot, dirs=dirs, rays=o, name=name)
    r.close()


def test_full_frame_rays_equal_emulation_of_oracle_weights(shipped):
    o = shipped["rays"]
    rgb, px = sv.sampling_view(o["oracle_weights"].cpu().numpy())
    _same(o["rgb"], rgb, "render_rays view vs the emulation of its d_oracle_weights")
    assert int(o["n_samples"].abs().sum()) == 0
    # the picture is not trivial: the sampling net spreads its leading cells over the frame
    assert len(np.unique(rgb[:, 0])) > 4


def test_full_frame_every_entry_draws_the_same_view(shipped):
    from test_stream_order import Surface
    r, thr, K, pose, rot = (shipped[k] for k in ("r", "thr", "K", "pose", "rot"))
    want_rgb = shipped["rays"]["rgb"].cpu().numpy()
    _, want_px = sv.sampling_view(shipped["rays"]["oracle_weights"].cpu().numpy())
    ns = r.render_camera(pose, rot, W, H, thr, K, want_nsamples=True)
    px = r.render_camera_rgba8(pose, rot, W, H, thr, K)
    surf = Surface(W, H)
    p, q = r._pose_rot(pose, rot)
    from adanerf_b200.renderer import _fptr
    r._check(r.lib.adn_render_camera_surface(r.handle, _fptr(p), _fptr(q), W, H, 0, H, float(thr), int(K), surf.surf.value,
                                             r._stream()))
    torch.cuda.synchronize()
    _same(ns["rgb"], want_rgb, "render_camera")
    assert int(ns["n_samples"].abs().sum()) == 0
    _same(px, want_px, "render_camera_rgba8 vs the quantised fp32 view")
    _same(surf.read().reshape(-1, 4), px, "surface vs rgba8")
    surf.free()
    hc = r.render_camera_host(pose, rot, W, H, thr, K, want_nsamples=True)
    _same(hc["rgb"], want_rgb, "render_camera_host")
    assert not hc["n_samples"].any()
    hr = r.render_rays_host(pose, rot, shipped["dirs"].cpu().numpy(), thr, K)
    _same(hr["rgb"], want_rgb, "render_rays_host")
    assert not hr["n_samples"].any()
    st = r.stats()
    assert st["n_samples"] == 0 and st["n_rays"] == W * H


def test_full_frame_chunks_and_row_bands_equal_the_whole_frame(shipped):
    r, thr, K, pose, rot = (shipped[k] for k in ("r", "thr", "K", "pose", "rot"))
    whole = r.render_camera_rgba8(pose, rot, W, H, thr, K).cpu().numpy()
    try:
        for chunk in (128, 1000, 77_777):
            r.set_option("chunk_rays", chunk)
            _same(r.render_camera_rgba8(pose, rot, W, H, thr, K), whole, f"chunk_rays {chunk}")
            o = r.render_rays(pose, rot, shipped["dirs"], thr, K)
            _same(o["rgb"], shipped["rays"]["rgb"], f"render_rays, chunk_rays {chunk}")
    finally:
        r.set_option("chunk_rays", 0)
    for row0, rows in ((0, 1), (1, 299), (300, 437), (737, 63)):
        band = r.render_camera_rgba8(pose, rot, W, H, thr, K, row0=row0, rows=rows)
        _same(band, whole[row0 * W:(row0 + rows) * W], f"rows {row0}..{row0 + rows}")


def test_full_frame_aux_outputs_are_refused(shipped):
    from adanerf_b200 import AdnError
    r = shipped["r"]
    with pytest.raises(AdnError) as e:
        r.render_rays(shipped["pose"], shipped["rot"], shipped["dirs"][:1000], shipped["thr"], shipped["K"], want_aux=("depth_map",))
    assert e.value.status == ADN_ERR_INVALID and "sampling_view" in str(e.value)


# ---- the option leaves normal renders alone -----------------------------------------------------------------------------------
def test_normal_render_is_unchanged_around_a_view_call(built, exports):
    from adanerf_b200 import Renderer
    r, thr, K = Renderer.from_export_dir(exports["pavillon_k16"])
    pose, rot = _pose_rot("pavillon_k16")
    before = r.render_camera_rgba8(pose, rot, W, H, thr, K).cpu().numpy()
    m_before = r.stats()["n_samples"]
    r.set_option("sampling_view", 1)
    view = r.render_camera_rgba8(pose, rot, W, H, thr, K).cpu().numpy()
    assert r.stats()["n_samples"] == 0
    r.set_option("sampling_view", 0)
    after = r.render_camera_rgba8(pose, rot, W, H, thr, K).cpu().numpy()
    _same(after, before, "normal render after a view call")
    assert r.stats()["n_samples"] == m_before > W * H
    assert not np.array_equal(view, before)
    r.close()


def test_budgeted_context_in_view_mode_renders_the_view_without_selection(built, exports, shipped):
    from adanerf_b200 import Renderer
    name = shipped["name"]
    r, thr, K = Renderer.from_export_dir(exports[name])
    pose, rot = shipped["pose"], shipped["rot"]
    r.set_option("sample_budget", W * H + 1000)
    r.set_option("sampling_view", 1)
    l0 = r.stats()["kernel_launches"]
    r.set_option("profile", 1)
    px = r.render_camera_rgba8(pose, rot, W, H, thr, K)
    st = r.stats()
    _, want = sv.sampling_view(shipped["rays"]["oracle_weights"].cpu().numpy())
    _same(px, want, "budgeted view")
    chunk = -(-max(8192, (8 << 20) // K) // 128) * 128              # the automatic chunk, in whole rows
    chunk = chunk if chunk % W == 0 else (chunk // W + 1) * W
    chunks = -(-W * H // chunk)
    assert st["kernel_launches"] - l0 == 3 * chunks          # stage 0, sampling MLP and the view per chunk: no selection
    assert st["n_samples"] == 0
    ms = st["ms_stage"]
    assert ms[0] > 0 and ms[1] > 0 and ms[5] > 0 and ms[2] == ms[3] == ms[4] == 0.0
    assert r.last_threshold() == np.float32(thr)
    r.close()


# ---- order -----------------------------------------------------------------------------------------------------------------------
def test_view_calls_stay_behind_an_earlier_call_on_a_held_stream(built, renderer):
    """A view render on a second stream, and the stage entry, wait for an earlier call held on a gated stream; a view render
    on a capturing stream is refused."""
    from test_stream_order import Gate
    from adanerf_b200 import AdnError
    from adanerf_b200.renderer import _fptr
    r = renderer
    scene = orc.SCENE_BARBERSHOP
    pose, rot = r._pose_rot(torch.tensor(scene["view_cell_center"]), torch.eye(3))
    n_rows, K, thr = 25, 8, 0.2
    gate = Gate()
    r.set_option("sampling_view", 1)
    try:
        def view_on(stream, out):
            r._check(r.lib.adn_render_camera_rgba8(r.handle, _fptr(pose), _fptr(rot), W, H, 300, n_rows, thr, K, out.data_ptr(),
                                                   C.c_void_p(stream.cuda_stream)))
        a_ref = torch.empty((n_rows * W, 4), dtype=torch.uint8, device="cuda")
        b_ref = torch.empty_like(a_ref)
        view_on(torch.cuda.current_stream(), a_ref)
        raw0 = r.mlp0(r.stage0(pose, rot, r.generate_ray_directions(W, H, 300, n_rows))[0])
        sv_ref = r.sampling_view(raw0)
        torch.cuda.synchronize()
        b_ref.copy_(a_ref)
        # a view render on s2 behind a call held on s1
        a, b = torch.zeros_like(a_ref), torch.zeros_like(a_ref)
        done = torch.cuda.Event()
        gate.shut(gate.s1.cuda_stream)
        view_on(gate.s1, a)
        view_on(gate.s2, b)
        done.record(gate.s2)
        time.sleep(0.3)
        ran_early = done.query()
        gate.open()
        torch.cuda.synchronize()
        assert not ran_early, "the view call on the second stream ran before the held call"
        _same(a, a_ref, "held call")
        _same(b, b_ref, "second-stream call")
        # the stage entry (the context's own stream) returns only after the held call has run
        gate.shut(gate.s1.cuda_stream)
        view_on(gate.s1, a)
        opened_at = {}

        def opener():
            time.sleep(0.5)
            opened_at["t"] = time.monotonic()
            gate.cu.cuCtxSetCurrent(gate.ctx)
            gate.open()
        t = threading.Thread(target=opener)
        t.start()
        out = r.sampling_view(raw0)
        returned = time.monotonic()
        t.join()
        torch.cuda.synchronize()
        assert returned >= opened_at["t"], "adn_sampling_view returned before the earlier call ran"
        _same(out["rgba8"], sv_ref["rgba8"], "stage entry behind a held call")
        # capture is refused
        s = gate.s2
        c = torch.zeros_like(a_ref)
        torch.cuda.synchronize()
        err = None
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            try:
                view_on(s, c)
            except AdnError as e:
                err = e
        del g
        assert err is not None and err.status == ADN_ERR_INVALID and "capturing a CUDA graph" in str(err)
        with torch.cuda.stream(s):
            view_on(s, c)
        torch.cuda.synchronize()
        _same(c, a_ref, "after the refused capture")
        # the stage entry synchronises, so it cannot be captured: refused before any CUDA call, and the capture survives
        err = None
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            try:
                r.sampling_view(raw0)
            except AdnError as e:
                err = e
        del g
        assert err is not None and err.status == ADN_ERR_INVALID and "capturing a CUDA graph" in str(err)
        _same(r.sampling_view(raw0)["rgba8"], sv_ref["rgba8"], "stage entry after the refused capture")
    finally:
        r.set_option("sampling_view", 0)
        gate._streams.destroy()


# ---- the headless viewer ---------------------------------------------------------------------------------------------------
def test_headless_viewer_oracle_surface(built, exports):
    r = subprocess.run([built.VIEWER, exports["barbershop_k4"], "--oracle", "--surface", "-f", "3"], capture_output=True, text=True,
                       timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert f"surface frame {W}x{H} (sampling view): 0 mismatching bytes" in r.stdout, r.stdout
    assert "last frame 0 samples" in r.stdout, r.stdout


def test_multi_gpu_view_applies_no_budget(built, exports, shipped):
    """adn_multi with the view on draws the single-context view and makes none of the frame budget's checks: a budget below
    the frame's rays, which a budgeted frame refuses, renders the view."""
    from adanerf_b200 import AdnError
    from adanerf_b200.multi import MultiRenderer, load_multi_library
    lib = load_multi_library()
    h, thr, K, dev = C.c_void_p(), C.c_float(), C.c_int(), (C.c_int * 1)(0)
    assert lib.adn_multi_create_from_export_dir(C.byref(h), exports[shipped["name"]].encode(), dev, 1, C.byref(thr), C.byref(K)) == 0
    m = MultiRenderer.__new__(MultiRenderer)                         # the binding over a handle made from the export directory
    m.lib, m.devices, m.handle, m._shape, m._issued, m._waited = lib, [0], h, [None, None], 0, 0
    try:
        m.set_option("sample_budget", 1000)
        with pytest.raises(AdnError):
            m.render_camera(shipped["pose"], shipped["rot"], W, H, shipped["thr"], shipped["K"])   # B < W * H
        m.set_option("sampling_view", 1)
        m.render_camera(shipped["pose"], shipped["rot"], W, H, shipped["thr"], shipped["K"])
        frame = m.wait_frame().cpu()
        _same(frame, shipped["rays"]["rgb"], "multi-GPU view under a budget")
        assert m.last_threshold() == np.float32(shipped["thr"])
    finally:
        m.close()


def _ppm(path):
    with open(path, "rb") as f:
        data = f.read()
    assert data.startswith(b"P6\n400 301\n255\n"), data[:20]
    return data


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
@pytest.mark.parametrize("budget", [[], ["--budget", "1000"]], ids=["no_budget", "budget_below_rays"])
def test_headless_viewer_oracle_on_two_gpus_equals_one(built, exports, budget):
    """The frame's pixels (-w), not only a checksum: a band in the wrong place would change them."""
    d = exports["pavillon_k16"]
    frame = os.path.join(d, "adn_frame.ppm")
    one = subprocess.run([built.VIEWER, d, "--oracle", "-s", "400", "301", "-f", "4", "-w"] + budget, capture_output=True, text=True,
                         timeout=300)
    assert one.returncode == 0, one.stdout + one.stderr
    px1 = _ppm(frame)
    os.remove(frame)
    two = subprocess.run([built.VIEWER, d, "--oracle", "-s", "400", "301", "-f", "4", "-g", "2", "-w"] + budget, capture_output=True,
                         text=True, timeout=300)
    assert two.returncode == 0, two.stdout + two.stderr
    px2 = _ppm(frame)
    assert px1 == px2, f"{sum(a != b for a, b in zip(px1, px2))} bytes of the 2-GPU frame differ from the 1-GPU frame"
    assert len(set(px1[20:])) > 4                                    # not a blank frame
