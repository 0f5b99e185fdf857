"""Positional encodings other than posEncArgs 10-4 (2-2 for the sampling net) on the H100: stage 0 and stage 3 on whole
800 x 800 frames against the fp32-faithful emulation (geometry bit for bit, sincosf anchors within 2 ulp, every recurrence
band equal to the emulated recurrence from the kernel's own anchors), the shading kernel bit for bit on exactly-summing
nets with one- and two-block position inputs, end-to-end parity with the oracle, the fused encoder, dense and
sample-budget renders, the export path, and rejections of weights that disagree with the scene."""
import re
import subprocess

import numpy as np
import pytest
import torch

from oracle import adanerf_oracle as orc
from oracle import shape_emulation as she
from oracle import stage_emulation as se
from test_encodings import CASES, bands, case_scene, case_weights, columns, exact_shading_net, mlp1_emulate, oracle_render
from conftest import load_golden
from oracle import gen_encoding_golden as geg
from test_mlp_kernel_exact import _first_difference, _row_counts
from test_net_shapes_gpu import _packed_mask

pytestmark = pytest.mark.gpu

W = H = 800
POSE_ROT = (torch.tensor([0.05, -0.03, 0.02]), orc.rotation_yaw(20.0))


def _renderer(scene, sd0=None, sd1=None):
    from adanerf_b200 import Renderer
    return Renderer(scene, device=0, sampling_net=sd0, shading_net=sd1)


def _pose(scene):
    return torch.tensor(scene["view_cell_center"], dtype=torch.float32) + POSE_ROT[0], POSE_ROT[1].reshape(3, 3)


def _ulps(a, b):
    ia = np.asarray(a, np.float32).view(np.int32).astype(np.int64)
    ib = np.asarray(b, np.float32).view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = np.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return np.abs(ia - ib)


def _check_encoding(got, v, L, what):
    """got [N, 3 + 6L]: the kernel's encoding of v [N, 3].  v itself bit for bit; the anchors (bands f % 5 == 0) within
    2 ulp of the correctly rounded sin / cos; every band equal to the recurrence emulated from the kernel's own anchors,
    and within recurrence_band_bounds of float64."""
    got = np.asarray(got, np.float32)
    assert got.shape[1] == 3 + 6 * L, what
    assert np.array_equal(got[:, :3].view(np.uint32), np.asarray(v, np.float32).view(np.uint32)), what + ": inputs"
    if L == 0:
        return
    exact = se.posenc3(v, L)
    for f in range(0, L, se.ANCHOR_EVERY):
        cols = slice(3 + 6 * f, 9 + 6 * f)
        assert int(_ulps(got[:, cols], exact[:, cols]).max()) <= 2, f"{what}: anchor band {f}"
    emu = se.posenc3(v, L, anchors=got)
    assert np.array_equal(got.view(np.uint32), emu.view(np.uint32)), what + ": recurrence bands"
    bound = se.recurrence_band_bounds(L=L)
    err = np.abs(got.astype(np.float64) - se.posenc_f64(v, L))[:, 3:].reshape(-1, L, 6).max(axis=(0, 2))
    assert np.all(err <= bound), (what, err, bound)


SAMPLING_ENCODINGS = [(16, 4), (-1, -1), (3, 2), (0, 9)]


@pytest.mark.parametrize("p0,d0", SAMPLING_ENCODINGS, ids=lambda v: str(v))
def test_stage0_on_a_full_frame(p0, d0):
    scene = dict(orc.SCENE_PAVILLON, n_freq_pos0=p0, n_freq_dir0=d0)
    (P0, D0), _ = bands(scene)
    r = _renderer(scene)
    try:
        pose, rot = _pose(scene)
        dirs = r.generate_ray_directions(W, H)
        x0, ro, rd = r.stage0(pose, rot, dirs)
        torch.cuda.synchronize()
        assert x0.shape[1] == columns(scene)[0] == 6 + 6 * (P0 + D0)
        p, nds, pd = se.stage0(pose.numpy(), rot.numpy(), dirs.cpu().numpy(), scene, nfd=0, nfp=0)   # pd = [dn, p]
        assert np.array_equal(ro.cpu().numpy().view(np.uint32), p.view(np.uint32))
        assert np.array_equal(rd.cpu().numpy().view(np.uint32), nds.view(np.uint32))
        x = x0.cpu().numpy()
        _check_encoding(x[:, :3 + 6 * D0], pd[:, :3], D0, "direction block")
        _check_encoding(x[:, 3 + 6 * D0:], p, P0, "position block")
    finally:
        r.close()


@pytest.mark.parametrize("name,fields,shape", CASES, ids=[c[0] for c in CASES])
def test_stage3_on_a_full_frame(name, fields, shape):
    scene = case_scene(fields)
    _, (P, D) = bands(scene)
    r = _renderer(scene)
    try:
        pose, rot = _pose(scene)
        _, ro, rd = r.stage0(pose, rot, r.generate_ray_directions(W, H))
        n = ro.shape[0]
        g = torch.Generator().manual_seed(3)
        ray = torch.randint(0, n, (4 * n,), generator=g, dtype=torch.int32)
        z = torch.from_numpy(se.zlut(scene))[torch.randint(0, 128, (4 * n,), generator=g)]
        x1 = r.stage3(ro, rd, ray.cuda(), z.cuda())
        torch.cuda.synchronize()
        assert x1.shape == (4 * n, (3 + 6 * P) + (3 + 6 * D))
        pos, d = se.sample_inputs(scene, ro.cpu().numpy(), rd.cpu().numpy(), ray.numpy(), z.numpy())
        x = x1.cpu().numpy()
        _check_encoding(x[:, :3 + 6 * P], pos, P, "position block")
        _check_encoding(x[:, 3 + 6 * P:], d, D, "view block")
    finally:
        r.close()


# --------------------------------------------------------------------------------------------------- MLP kernels
@pytest.mark.parametrize("n_p,n_v", [(39, 15), (123, 63), (3, 3)], ids=["P39-V15", "P123-V63", "none"])
@pytest.mark.parametrize("shape", [(8, 256, 4), (6, 128, 3), (4, 128, -1), (2, 256, 0)], ids=lambda s: "x".join(map(str, s)))
def test_mlp1_bit_exact(shape, n_p, n_v):
    rows = _row_counts()
    sd, x = exact_shading_net(shape, n_p, n_v, rows=rows[-1], device="cuda")
    r = _renderer(dict(orc.SCENE_PAVILLON, n_freq_pos=(n_p - 3) // 6 or -1, n_freq_dir=(n_v - 3) // 6 or -1,
                       n_freq_pos0=10, n_freq_dir0=4))
    try:
        r.set_weights(1, sd)
        assert r.net_shape(1) == shape and r.net_dims(1) == (n_p + n_v, 4)
        ref = mlp1_emulate(x, sd, n_p)
        for n in rows:
            out = r.mlp1(x[:n])
            assert torch.equal(out, ref[:n]), f"{n} rows: " + _first_difference(out, ref[:n])
    finally:
        r.close()


@pytest.mark.parametrize("n_in", [6, 126])
def test_mlp0_bit_exact_at_the_sampling_limits(n_in):
    rows = _row_counts()
    sd, x = she.exact_sampling_net(n_in, 6, 128, 3, rows=rows[-1], device="cuda", width=128)
    from oracle import mlp_emulation as me
    r = _renderer(orc.SCENE_PAVILLON)
    try:
        r.set_weights(0, sd)
        ref = me.mlp0_emulate(x, sd, terms=3)
        for n in rows:
            out = r.mlp0(x[:n])
            assert torch.equal(out, ref[:n]), f"{n} rows: " + _first_difference(out, ref[:n])
    finally:
        r.close()


# ------------------------------------------------------------------------------------------ end to end, each case
@pytest.mark.parametrize("name,fields,shape", CASES, ids=[c[0] for c in CASES])
def test_parity_with_the_oracle(name, fields, shape):
    scene = case_scene(fields)
    thr, K = (0.15, 16) if fields.get("use_ndc") else (0.2, 8)
    sd0, sd1 = case_weights(scene, shape)
    r = _renderer(scene, sd0, sd1)
    try:
        pose, rot = _pose(scene)
        dirs = r.generate_ray_directions(W, H)[::16].contiguous()
        out = r.render_rays(pose, rot, dirs, thr, K)
        ref = oracle_render(pose, rot, dirs.cpu(), sd0, sd1, scene, thr, K)
        same = float((out["n_samples"].cpu().long() == ref["n_samples"]).double().mean())
        psnr = orc.psnr(out["rgb"].cpu().clamp(0, 1), ref["rgb"].clamp(0, 1))
        print(f"{name}: {dirs.shape[0]} rays, identical sample counts on {100 * same:.3f} %, PSNR against the oracle {psnr:.2f} dB")
        assert same >= 0.999 and psnr >= 49.4   # |dPSNR| < 0.05 dB for a 30 dB scene (test_parity_gate.py)
        # the fused encoder computes the same tiles as stage 3 (non-NDC scenes; NDC always runs stage 3)
        full = r.render_camera(pose, rot, W, H, thr, K)["rgb"]
        r.set_option("fuse_encoder", 1)
        fused = r.render_camera(pose, rot, W, H, thr, K)["rgb"]
        r.set_option("fuse_encoder", 0)
        assert torch.equal(full, fused)
        # render_camera renders what render_rays renders for the same rays
        assert torch.equal(full[::16], out["rgb"])
    finally:
        r.close()


def test_dense_and_sample_budget_on_a_two_block_encoding():
    name, fields, shape = CASES[0]
    scene = case_scene(fields)
    sd0, sd1 = case_weights(scene, shape)
    r = _renderer(scene, sd0, sd1)
    try:
        pose, rot = _pose(scene)
        d = r.generate_ray_directions(W, H)
        dirs = d[::400].contiguous()
        out = r.render_rays(pose, rot, dirs, 0.0, 128)
        ref = oracle_render(pose, rot, dirs.cpu(), sd0, sd1, scene, 0.0, 128)
        scale = max(1.0, float(ref["rgb"].abs().max()))   # dense zp = raw0 puts these colours outside [0, 1]
        psnr = orc.psnr(out["rgb"].cpu() / scale, ref["rgb"] / scale)
        print(f"dense K=128: PSNR against the oracle {psnr:.2f} dB at scale {scale:.3g}")
        assert torch.isfinite(out["rgb"]).all() and torch.equal(out["n_samples"].cpu().long(), ref["n_samples"]) and psnr >= 49.4
        r.set_option("fuse_encoder", 1)
        assert torch.equal(r.render_rays(pose, rot, dirs, 0.0, 128)["rgb"], out["rgb"])
        r.set_option("fuse_encoder", 0)
        free = r.render_rays(pose, rot, d, 0.1, 8)
        budget = int(free["n_samples"].sum()) // 2
        r.set_option("sample_budget", budget)
        got = r.render_rays(pose, rot, d, 0.1, 8)
        t = r.last_threshold()
        r.set_option("sample_budget", 0)
        fixed = r.render_rays(pose, rot, d, t, 8)
        assert int(got["n_samples"].sum()) <= budget
        assert torch.equal(got["rgb"], fixed["rgb"]) and torch.equal(got["n_samples"], fixed["n_samples"])
    finally:
        r.close()


# ------------------------------------------------------------------------------------------------ export path
@pytest.mark.parametrize("fields,pos_enc,args", [
    (dict(n_freq_pos=20, n_freq_dir=10, n_freq_pos0=-1, n_freq_dir0=-1), "[none, nerf]", "[10-4, 20-10]"),
    (dict(n_freq_pos=6, n_freq_dir=2, n_freq_pos0=16, n_freq_dir0=4), "[nerf, nerf]", "[16-4, 6-2]"),
], ids=["none-20-10", "16-4-6-2"])
def test_export_dir_and_viewer(tmp_path, fields, pos_enc, args):
    import __graft_entry__ as g
    from adanerf_b200 import Renderer
    from adanerf_b200 import onnx_weights as ow
    scene = case_scene(fields)
    sd0, sd1 = case_weights(scene, (8, 256, 4))
    d = tmp_path / "export"
    ow.write_export_dir(str(d), scene, sd0, sd1, 0.2, 8)
    cfg = (d / "config.ini").read_text()
    assert f"posEnc = {pos_enc}\n" in cfg and f"posEncArgs = {args}\n" in cfg
    r1, thr, K = Renderer.from_export_dir(str(d))
    r2 = _renderer(scene, sd0, sd1)
    try:
        pose, rot = _pose(scene)
        a = r1.render_camera(pose, rot, 200, 200, thr, K)["rgb"]
        b = r2.render_camera(pose, rot, 200, 200, 0.2, 8)["rgb"]
        assert torch.equal(a, b)
        assert r1.n_feat0 == columns(scene)[0] and r1.n_feat1 == sum(columns(scene)[1:])
        x0, _, _ = r1.stage0(pose, rot, r1.generate_ray_directions(8, 8))
        assert x0.shape[1] == columns(scene)[0]
    finally:
        r1.close()
        r2.close()
    res = subprocess.run([g.VIEWER, str(d), "-s", "400", "300", "-f", "2"], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stdout + res.stderr
    (p0, d0), (p, dd) = bands(scene)
    enc0 = "none" if fields["n_freq_pos0"] < 0 else f"{p0}-{d0}"
    assert f"net 0: sampling 8 x 256, skip -1, posEnc {enc0}" in res.stdout, res.stdout
    assert f"net 1: shading 8 x 256, skip 4, posEnc {p}-{dd}" in res.stdout, res.stdout
    assert re.search(r"2 frames 400x300: ([0-9.]+) ms/frame", res.stdout), res.stdout


# ------------------------------------------------------------------------------------------------ rejections
def test_weights_that_disagree_with_the_scene_are_rejected():
    from adanerf_b200 import AdnError
    scene = case_scene(CASES[0][1])   # shading 20-10: P = 123, V = 63
    r = _renderer(scene)
    try:
        sd = orc.init_shading_net()   # a 10-4 net
        with pytest.raises(AdnError) as e:
            r.set_weights(1, sd)
        assert e.value.status == 1 and "pts_linears.0.weight must be [W, 123] (posEnc 20-10)" in str(e.value), str(e.value)
        _, sd = case_weights(scene, (8, 256, 4))
        sd["views_linears.0.weight"] = torch.zeros(128, 256 + 27)
        with pytest.raises(AdnError) as e:
            r.set_weights(1, sd)
        assert "views_linears.0.weight must be [128, 319]" in str(e.value), str(e.value)
    finally:
        r.close()
    with pytest.raises(AdnError) as e:   # outside the tile formats
        _renderer(dict(orc.SCENE_PAVILLON, n_freq_pos=21))
    assert e.value.status == 1
    with pytest.raises(AdnError):
        _renderer(dict(orc.SCENE_PAVILLON, n_freq_pos0=16, n_freq_dir0=5))


# ---------------------------------------------------------------------------------- the reference's own outputs
@pytest.mark.parametrize("name", list(geg.CASES))
def test_encoding_golden_parity_gate(name):
    """The reference's outputs for the case (tests/golden/enc_*, oracle/gen_encoding_golden.py): identical sample counts
    on >= 99.9 % of the rays, PSNR >= 49.4 dB (|dPSNR| < 0.05 dB for a 30 dB scene), the sampling net's raw0 and stage 0's
    features and rays against the reference's, and stage 2 on the reference's raw0 selects and compacts exactly the
    reference's samples."""
    g = load_golden(name)
    m = g["meta"]
    scene = m["scene_params"]
    sd0, sd1 = geg.case_weights(name)
    r = _renderer(scene, sd0, sd1)
    try:
        pose, rot = torch.from_numpy(g["pose"]), torch.from_numpy(g["rot"])
        dirs = torch.from_numpy(g["dirs"]).cuda()
        for fused in (0, 1):
            r.set_option("fuse_encoder", fused)
            out = r.render_rays(pose, rot, dirs, m["thr"], m["K"], want_oracle_weights=True)
            same = (out["n_samples"].cpu().numpy() == np.round(g["asp"] * m["K"]).astype(np.int32)).mean()
            p = orc.psnr(out["rgb"].cpu().numpy(), g["rgb"])
            print(f"{name} fuse_encoder {fused}: identical counts {same:.4f}, PSNR(ours, reference) {p:.2f} dB")
            assert same >= 0.999 and p >= 49.4
        r.set_option("fuse_encoder", 0)
        np.testing.assert_allclose(out["oracle_weights"].cpu().numpy(), g["raw0"], rtol=0, atol=2e-4 * max(1, np.abs(g["raw0"]).max()))
        x0, ro, rd = r.stage0(pose, rot, dirs)
        np.testing.assert_allclose(x0.cpu().numpy(), g["x0"], rtol=0, atol=2e-5)
        np.testing.assert_allclose(ro.cpu().numpy(), g["ray_o"], rtol=0, atol=1e-6)
        s2 = r.stage2(torch.from_numpy(g["raw0"]).cuda(), m["thr"], m["K"])
        mask = _packed_mask(g)
        np.testing.assert_array_equal(s2["count"].cpu().numpy(), mask.sum(1))
        np.testing.assert_array_equal(s2["ray"].cpu().numpy(), np.nonzero(mask)[0])
        # stage 3 on the reference's samples of the first rays against the reference's features
        x1 = g["x1_nan"]
        live = np.isfinite(x1[..., 0])
        n1 = int(live.sum())
        got = r.stage3(ro, rd, s2["ray"][:n1], s2["z"][:n1]).cpu().numpy()
        # band f reads the argument 2^f v: an ulp of difference in v between two fp32 evaluations of the sample position
        # (~6e-8 for |v| ~ 1) moves it by 2^f ulps, so the tolerance grows with the band (SURVEY 8d: 5e-4 at 2^9)
        _, (P, D) = bands(scene)
        band_tol = lambda L: np.concatenate([[5e-4] * 3] + [[max(5e-4, 1e-7 * 2.0 ** f)] * 6 for f in range(L)])
        err = np.abs(got.astype(np.float64) - x1[live]) - np.concatenate([band_tol(P), band_tol(D)])
        assert float(err.max()) <= 0.0, f"column {int(err.max(0).argmax())}: {float(err.max()):.3g} past its tolerance"
    finally:
        r.close()


def test_export_with_a_zero_sampling_band_count_renders(tmp_path):
    """posEncArgs [0-4, 10-4]: the loader reads the sampling net's 0 position bands as zero bands (30 columns), so the
    export renders what its state dicts render."""
    from adanerf_b200 import Renderer
    from adanerf_b200 import onnx_weights as ow
    scene = dict(orc.SCENE_PAVILLON, n_freq_pos0=-1, n_freq_dir0=4)
    torch.manual_seed(0)
    sd0, sd1 = orc.init_sampling_net(n_in=30), orc.init_shading_net()
    sd0["layers.7.weight"] = sd0["layers.7.weight"] * 0.15
    ow.write_export_dir(str(tmp_path), scene, sd0, sd1, 0.2, 8)
    r1, thr, K = Renderer.from_export_dir(str(tmp_path))
    r2 = _renderer(scene, sd0, sd1)
    try:
        assert r1.n_feat0 == 30
        pose, rot = _pose(scene)
        assert torch.equal(r1.render_camera(pose, rot, 200, 200, thr, K)["rgb"], r2.render_camera(pose, rot, 200, 200, 0.2, 8)["rgb"])
    finally:
        r1.close()
        r2.close()
