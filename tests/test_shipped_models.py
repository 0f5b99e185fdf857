"""The reference's two shipped trained models, from their own export directories (tests/golden/shipped/, byte-for-byte
copies written by oracle/gen_shipped_golden.py): Barbershop (adanerf_real_time_viewer/sample, K = 4, thr 0.15, the
viewer's default model) and Pavillon (sample_pavillon_16, K = 16, thr 0.15).  The model files are the ones
torch.onnx.export wrote, not re-encoded, so the C++ loader and the Python reader are tested on that byte layout; the
renders are tested against the reference's own stages (barber_* goldens) and against the CPU oracle on full frames."""
import ctypes as C
import hashlib
import json
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from conftest import GOLDEN, load_golden, load_pavillon_weights
from adanerf_b200 import onnx_weights as ow
from adanerf_b200.convert import read_dataset_info
from adanerf_b200.synthetic import load_weights_npz
from oracle import adanerf_oracle as orc

SHIPPED = {"barbershop_k4": (orc.SCENE_BARBERSHOP, 4, 0.15), "pavillon_k16": (orc.SCENE_PAVILLON, 16, 0.15)}
BARBER_CASES = ["barber_k4_t0.15", "barber_k16_t0.5"]
SCENE_KEYS = ("view_cell_center", "view_cell_size", "depth_range", "fov", "max_depth")
NET_SHAPES = ((8, 256, -1), (8, 256, 4))
PART_BYTES = 1_000_000
W = H = 800
RX = torch.tensor([[1, 0, 0], [0, 0, -1], [0, 1, 0]], dtype=torch.float32)   # camera -z -> world +y
# two poses inside each view cell, neither at its centre, looking along the floor in different directions
POSES = {"barbershop_k4": [([0.3, -0.2, 0.08], 35.0), ([-0.5, 0.45, -0.15], 200.0)],
         "pavillon_k16": [([0.05, -0.03, 0.02], 0.0), ([-0.2, 0.25, -0.06], 120.0)]}


def load_barbershop_weights():
    """(sampling, shading) state_dicts of the shipped Barbershop networks (tests/golden/weights_barbershop)."""
    return load_weights_npz(os.path.join(GOLDEN, "weights_barbershop"))


def shipped_weights(name):
    return load_barbershop_weights() if name.startswith("barber") else load_pavillon_weights()


def pose_rot(name, i):
    off, yaw = POSES[name][i]
    scene = SHIPPED[name][0]
    return torch.tensor(scene["view_cell_center"]) + torch.tensor(off), orc.rotation_yaw(yaw) @ RX


def _bits(a):
    return np.asarray(a, dtype=np.float32).view(np.uint32)


@pytest.fixture(scope="module")
def export_dirs(tmp_path_factory):
    """name -> (the shipped export directory reassembled from its parts, its manifest)."""
    out = {}
    for name in SHIPPED:
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
        out[name] = (str(dst), man)
    return out


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    from adanerf_b200 import load_library
    return load_library()


# ------------------------------------------------------------------------------------------------------------ CPU
def test_reassembled_files_match_the_manifest(export_dirs):
    for name, (d, man) in export_dirs.items():
        assert sorted(man["files"]) == ["config.ini", "dataset_info.txt", "model0.onnx", "model1.onnx"]
        for fname, e in man["files"].items():
            data = open(os.path.join(d, fname), "rb").read()
            assert len(data) == e["size"] and hashlib.sha256(data).hexdigest() == e["sha256"], (name, fname)
            for p in e.get("parts", []):
                assert os.path.getsize(os.path.join(GOLDEN, "shipped", name, p)) <= PART_BYTES
    # the two configs are the two forms the reference ships: the full training config and a minimal one
    assert os.path.getsize(os.path.join(export_dirs["barbershop_k4"][0], "config.ini")) == 2192
    assert os.path.getsize(os.path.join(export_dirs["pavillon_k16"][0], "config.ini")) == 609


@pytest.mark.parametrize("name", list(SHIPPED))
def test_probe_reads_the_shipped_export_dir(name, lib, export_dirs):
    """adn_probe_export_dir on the reference's own files: K, thr, the initialiser counts of the two networks, and every
    scene parameter equal, bit for bit, to float32 of what the Python parser reads from dataset_info.txt."""
    from adanerf_b200._lib import Scene
    d, _ = export_dirs[name]
    scene, K, thr = SHIPPED[name]
    sc, t, k, n = Scene(), C.c_float(), C.c_int(), (C.c_int * 2)()
    assert lib.adn_probe_export_dir(d.encode(), C.byref(sc), C.byref(t), C.byref(k), n) == 0
    assert k.value == K and _bits(t.value) == _bits(thr) and list(n) == [16, 24]
    info = read_dataset_info(os.path.join(d, "dataset_info.txt"))
    for key in SCENE_KEYS:
        got = getattr(sc, key)
        got = list(got) if key in ("view_cell_center", "view_cell_size", "depth_range") else [got]
        want = info[key] if isinstance(info[key], list) else [info[key]]
        np.testing.assert_array_equal(_bits(got), _bits(want), err_msg=key)
        np.testing.assert_array_equal(_bits(want), _bits(np.atleast_1d(scene[key])), err_msg=key)
    assert (sc.use_ndc, sc.n_freq_pos, sc.n_freq_dir) == (0, 10, 4)


@pytest.mark.parametrize("name", list(SHIPPED))
def test_python_reader_on_the_shipped_models(name, export_dirs):
    """onnx_weights.read_onnx_initializers on the files torch.onnx.export wrote equals the stored weights bit for bit."""
    d, _ = export_dirs[name]
    sds = shipped_weights(name)
    for i in range(2):
        back = ow.read_onnx_initializers(os.path.join(d, f"model{i}.onnx"))
        assert sorted(back) == sorted(sds[i])
        for k, v in back.items():
            assert v.dtype == np.float32 and v.shape == tuple(sds[i][k].shape), k
            np.testing.assert_array_equal(v.view(np.uint32), sds[i][k].numpy().view(np.uint32), err_msg=k)
    assert ow.net_shapes(*sds) == NET_SHAPES


def _oracle_run(case):
    g = load_golden(case)
    m = g["meta"]
    sd0, sd1 = load_barbershop_weights()
    out = orc.render_rays(torch.from_numpy(g["pose"]), torch.from_numpy(g["rot"]), torch.from_numpy(g["dirs"]),
                          sd0, sd1, m["scene_params"], m["thr"], m["K"], return_stages=True)
    return g, m, out


@pytest.mark.parametrize("case", BARBER_CASES)
def test_oracle_reproduces_the_barber_goldens(case):
    """The checks of tests/test_oracle_golden.py on the reference's stages for the trained Barbershop networks."""
    g, m, o = _oracle_run(case)
    np.testing.assert_array_equal(o["ray_d"].numpy(), g["ray_d"])
    np.testing.assert_allclose(o["ray_o"].numpy(), g["ray_o"], rtol=0, atol=1e-6)
    np.testing.assert_allclose(o["x0"].numpy(), g["x0"], rtol=0, atol=2e-4)
    s2 = orc.stage2_sample(torch.from_numpy(g["raw0"]), m["thr"], m["K"], m["scene_params"]["depth_range"])
    z = s2["z"].numpy().copy()
    z[~np.isfinite(z)] = np.nan
    np.testing.assert_array_equal(z, g["z_nan"])
    np.testing.assert_array_equal((s2["count"].numpy() / m["K"]).astype(np.float32), g["asp"])
    np.testing.assert_allclose(o["raw0"].numpy(), g["raw0"], rtol=0, atol=5e-4)
    same = (o["asp"].numpy() == g["asp"])
    assert same.mean() > 0.98
    assert np.abs(o["rgb"].numpy() - g["rgb"])[same].max() < 2e-3
    assert orc.psnr(o["rgb"].numpy()[same], g["rgb"][same]) > 60.0


# ------------------------------------------------------------------------------------------------------------ GPU
def _renderer(scene, sd0, sd1):
    from adanerf_b200 import Renderer
    return Renderer(scene, device=0, sampling_net=sd0, shading_net=sd1)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SHIPPED))
def test_loader_renders_like_the_state_dicts(name, export_dirs):
    """Renderer.from_export_dir (the C++ loader on the reference's files) == Renderer(scene, state dicts from the Python
    reader), bit for bit, at the shipped (thr, K)."""
    from adanerf_b200 import Renderer
    d, _ = export_dirs[name]
    _, K, thr = SHIPPED[name]
    r1, t1, k1 = Renderer.from_export_dir(d)
    scene = read_dataset_info(os.path.join(d, "dataset_info.txt"))
    sd0, sd1 = (ow.read_onnx_initializers(os.path.join(d, f"model{i}.onnx")) for i in range(2))
    r2 = _renderer(scene, sd0, sd1)
    try:
        assert k1 == K and _bits(t1) == _bits(thr)
        for r in (r1, r2):
            assert (r.net_shape(0), r.net_shape(1)) == NET_SHAPES and (r.n_feat0, r.n_feat1) == (90, 90)
        pose, rot = pose_rot(name, 0)
        a = r1.render_camera(pose, rot, W, H, t1, k1, want_nsamples=True)
        b = r2.render_camera(pose, rot, W, H, thr, K, want_nsamples=True)
        assert torch.isfinite(a["rgb"]).all()
        assert torch.equal(a["rgb"], b["rgb"]) and torch.equal(a["n_samples"], b["n_samples"])
        assert 1 <= int(a["n_samples"].min()) and int(a["n_samples"].max()) <= K
    finally:
        r1.close()
        r2.close()


@pytest.mark.gpu
@pytest.mark.parametrize("case", BARBER_CASES)
def test_barber_goldens_meet_the_budget(case):
    """The reference's outputs for the trained Barbershop networks: identical sample counts on >= 99.9 % of the rays,
    PSNR >= 49.4 dB, raw0 against the reference's, and stage 2 on the reference's raw0 compacts exactly the reference's
    samples."""
    g = load_golden(case)
    m = g["meta"]
    K = m["K"]
    sd0, sd1 = load_barbershop_weights()
    r = _renderer(m["scene_params"], sd0, sd1)
    try:
        pose, rot, dirs = torch.from_numpy(g["pose"]), torch.from_numpy(g["rot"]), torch.from_numpy(g["dirs"]).cuda()
        for fused in (0, 1):
            r.set_option("fuse_encoder", fused)
            out = r.render_rays(pose, rot, dirs, m["thr"], K, want_oracle_weights=True)
            same = (out["n_samples"].cpu().numpy() == np.round(g["asp"] * K).astype(np.int32)).mean()
            p = orc.psnr(out["rgb"].cpu().numpy(), g["rgb"])
            print(f"{case} fuse_encoder {fused}: identical counts {same:.4f}, PSNR(ours, reference) {p:.2f} dB")
            assert same >= 0.999 and p >= 49.4
            np.testing.assert_allclose(out["oracle_weights"].cpu().numpy(), g["raw0"], rtol=0,
                                       atol=2e-4 * max(1, np.abs(g["raw0"]).max()))
        r.set_option("fuse_encoder", 0)
        s2 = r.stage2(torch.from_numpy(g["raw0"]).cuda(), m["thr"], K)
        mask = np.isfinite(g["z_nan"])
        cnt = mask.sum(1)
        np.testing.assert_array_equal(s2["count"].cpu().numpy(), cnt)
        np.testing.assert_array_equal(s2["offset"].cpu().numpy(), np.concatenate([[0], np.cumsum(cnt)[:-1]]))
        np.testing.assert_array_equal(s2["ray"].cpu().numpy(), np.nonzero(mask)[0])
        o2 = orc.stage2_sample(torch.from_numpy(g["raw0"]), m["thr"], K, m["scene_params"]["depth_range"])
        np.testing.assert_array_equal(s2["cell"].cpu().numpy(), o2["cell"].numpy()[mask])
        np.testing.assert_array_equal(s2["zp"].cpu().numpy(), o2["zp"].numpy()[mask])
        # z = (w - 1) + d0 with w = (d1 - d0 + 1)^cell-centre: the library's table rounds the pow differently from the
        # reference's fp32 torch.pow (by one ulp of w in 19 of the 128 cells here), and with Barbershop's d0 < 0 the
        # subtraction cancels, so the bound is in ulps of w, not relative to z
        z_ref = g["z_nan"][mask]
        w = z_ref - np.float32(m["scene_params"]["depth_range"][0]) + np.float32(1)
        assert (np.abs(s2["z"].cpu().numpy() - z_ref) <= 2 * np.spacing(w)).all()
    finally:
        r.close()


@pytest.mark.gpu
@pytest.mark.parametrize("pose_i", [0, 1])
@pytest.mark.parametrize("name", list(SHIPPED))
def test_full_frame_at_the_shipped_setting_against_oracle(name, pose_i):
    """tests/test_parity_gate.py's full-frame gate at each model's shipped (thr, K): every ray of an 800 x 800 frame
    against the CPU oracle -- identical counts on >= 99.9 % of the rays, at most 0.1 % of the count histogram moved, PSNR
    >= 49.4 dB."""
    scene, K, thr = SHIPPED[name]
    sd0, sd1 = shipped_weights(name)
    pose, rot = pose_rot(name, pose_i)
    dirs = torch.from_numpy(orc.generate_ray_directions(W, H, scene["fov"]).reshape(-1, 3)).float()
    ref_rgb, ref_n = orc.render_frame(pose, rot, dirs, sd0, sd1, scene, thr, K)
    r = _renderer(scene, sd0, sd1)
    try:
        out = r.render_rays(pose, rot, dirs.cuda(), thr, K)
        rgb, n = out["rgb"].cpu(), out["n_samples"].cpu().long()
        same = (n == ref_n).float().mean().item()
        p = orc.psnr(rgb, ref_rgb)
        moved = int((torch.bincount(n, minlength=K + 1) - torch.bincount(ref_n, minlength=K + 1)).abs().sum()) // 2
        print(f"{name} pose {pose_i}: mean samples/ray {ref_n.float().mean():.3f}, rays with identical count {same:.6f} "
              f"({int((n != ref_n).sum())} differ, histogram mass moved {moved}), PSNR(ours, oracle) {p:.2f} dB")
        assert torch.isfinite(rgb).all()
        assert same >= 0.999
        assert moved <= 0.001 * W * H
        assert p >= 49.4
    finally:
        r.close()


@pytest.mark.gpu
def test_barbershop_delta_psnr_against_common_pseudo_ground_truth():
    """|dPSNR| < 0.05 dB as literally stated, at the shipped K = 4 / thr 0.15: PSNR of ours and of the oracle against a
    common image, the oracle's render at twice the samples and half the threshold (K 8, thr 0.075), on every 7th ray."""
    scene, K, thr = SHIPPED["barbershop_k4"]
    sd0, sd1 = load_barbershop_weights()
    pose, rot = pose_rot("barbershop_k4", 0)
    dirs = torch.from_numpy(orc.generate_ray_directions(W, H, scene["fov"]).reshape(-1, 3)).float()[::7].contiguous()
    gt = orc.render_rays(pose, rot, dirs, sd0, sd1, scene, thr / 2, 2 * K)["rgb"].clamp(0, 1)
    ref = orc.render_rays(pose, rot, dirs, sd0, sd1, scene, thr, K)["rgb"].clamp(0, 1)
    r = _renderer(scene, sd0, sd1)
    try:
        ours = r.render_rays(pose, rot, dirs.cuda(), thr, K)["rgb"].cpu().clamp(0, 1)
    finally:
        r.close()
    p_ref, p_ours = orc.psnr(ref, gt), orc.psnr(ours, gt)
    print(f"Barbershop PSNR vs pseudo ground truth: reference {p_ref:.3f} dB, ours {p_ours:.3f} dB, "
          f"delta {p_ours - p_ref:+.4f} dB; PSNR(ours, reference) {orc.psnr(ours, ref):.2f} dB")
    assert 15.0 < p_ref < 60.0
    assert abs(p_ours - p_ref) < 0.05


@pytest.mark.gpu
def test_barbershop_modes_at_k4():
    """At K = 4 with the trained networks: the render equals the stage entry points composed by hand at fuse_encoder 1
    and 0, bit for bit; under a sample budget of half the free frame's samples beyond one per ray, M <= B, the picture
    equals the fixed-threshold render at last_threshold(), and that threshold is budget_threshold of the frame's raw0."""
    from test_mlp_kernel_exact import _compose
    from test_sample_budget_oracle import budget_threshold
    scene, K, thr = SHIPPED["barbershop_k4"]
    sd0, sd1 = load_barbershop_weights()
    pose, rot = pose_rot("barbershop_k4", 1)
    r = _renderer(scene, sd0, sd1)
    try:
        dirs = r.generate_ray_directions(W, H)
        ref = _compose(r, pose, rot, dirs, thr, K)
        for fuse in (1, 0):
            r.set_option("fuse_encoder", fuse)
            out = r.render_rays(pose, rot, dirs, thr, K, want_oracle_weights=True)
            assert torch.equal(out["oracle_weights"], ref["raw0"]), fuse
            assert torch.equal(out["n_samples"], ref["n_samples"]), fuse
            assert torch.equal(out["rgb"], ref["rgb"]), fuse
            cam = r.render_camera(pose, rot, W, H, thr, K, want_nsamples=True)
            assert torch.equal(cam["rgb"], ref["rgb"]) and torch.equal(cam["n_samples"], ref["n_samples"]), fuse
        n = W * H
        free = int(ref["n_samples"].long().sum())
        B = n + (free - n) // 2
        r.set_option("sample_budget", B)
        out = r.render_rays(pose, rot, dirs, thr, K, want_oracle_weights=True)
        t = r.last_threshold()
        r.set_option("sample_budget", 0)
        fixed = r.render_rays(pose, rot, dirs, t, K)
        m = int(out["n_samples"].long().sum())
        print(f"Barbershop K=4: free frame {free} samples, budget {B}, t* = {t:.7g}, M = {m}")
        assert thr < t and m <= B
        assert _bits(t) == _bits(budget_threshold(out["oracle_weights"].cpu(), thr, K, B))
        assert torch.equal(out["rgb"], fixed["rgb"]) and torch.equal(out["n_samples"], fixed["n_samples"])
    finally:
        r.close()


@pytest.mark.gpu
def test_viewer_renders_the_shipped_barbershop(export_dirs):
    """The headless viewer on the reference's own default model directory, through the surface-object frame path."""
    import __graft_entry__ as g
    g.build()
    d, _ = export_dirs["barbershop_k4"]
    r = subprocess.run([g.VIEWER, d, "-s", str(W), str(H), "-f", "2", "--surface"], capture_output=True, text=True,
                       timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "K = 4," in r.stdout, r.stdout
    assert "net 0: sampling 8 x 256, skip -1, posEnc 10-4" in r.stdout, r.stdout
    assert "net 1: shading 8 x 256, skip 4, posEnc 10-4" in r.stdout, r.stdout
    assert f"surface frame {W}x{H}: 0 mismatching bytes" in r.stdout, r.stdout
    m = re.search(r"\(([0-9.]+) per ray\)", r.stdout)
    assert m and 1.0 <= float(m.group(1)) <= 4.0, r.stdout
