"""Networks of other depths, widths and skip positions than 8 x 256 / skip 4 on the H100: both MLP kernels bit for bit
against the emulation on exact networks, row by row on a full frame, the parity gate on the reference's own outputs for
such networks (tests/golden/shape_*), the fused encoder, dense and sample-budget renders, the export path and the
rejection of every unsupported shape."""
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import adanerf_oracle as orc
from oracle import mlp_emulation as me
from oracle import shape_emulation as se
from oracle import shape_oracle as so
from oracle.gen_shape_golden import CASES as SHAPE_CASES
from test_mlp_kernel_exact import FRAME_BOUNDS, _compose, _first_difference, _row_counts
from test_net_shapes import SHAPES, shape_case_weights, unsupported_nets

pytestmark = pytest.mark.gpu

W = H = 800


def _renderer(scene, sd0=None, sd1=None):
    from adanerf_b200 import Renderer
    return Renderer(scene, device=0, sampling_net=sd0, shading_net=sd1)


@pytest.fixture(scope="module")
def bare():
    r = _renderer(orc.SCENE_BARBERSHOP)
    yield r
    r.close()


@pytest.fixture
def make_renderer():
    made = []

    def make(scene, sd0=None, sd1=None):
        made.append(_renderer(scene, sd0, sd1))
        return made[-1]
    yield make
    for r in made:
        r.close()


def _skip_entry(shape):
    """make_shape_weights' skip argument that builds a shading net of shape (D, W, skip)."""
    D, _, skip = shape
    return "auto" if skip == 4 or (skip < 0 and D <= 4) else str(skip if skip >= 0 else D)


# ------------------------------------------------------------------------------------------------ bit-exact wiring
@pytest.mark.parametrize("terms", [3, 1])
@pytest.mark.parametrize("shape", se.EXACT_SAMPLING_SHAPES_W128, ids=lambda s: "x".join(map(str, s)))
def test_mlp0_bit_exact_on_w128_nets(bare, shape, terms):
    n_in, depth, n_out, width = shape
    rows = _row_counts()
    sd, x = se.exact_sampling_net(n_in, depth, n_out, terms, rows=rows[-1], device="cuda", width=width)
    bare.set_option("mlp0_terms", terms)
    try:
        bare.set_weights(0, sd)
        assert bare.net_shape(0) == (depth, width if depth > 1 else n_out, -1)
        ref = me.mlp0_emulate(x, sd, terms=terms)
        for n in rows:
            out = bare.mlp0(x[:n])
            assert torch.equal(out, ref[:n]), f"{n} rows: " + _first_difference(out, ref[:n])
    finally:
        bare.set_option("mlp0_terms", 3)


@pytest.mark.parametrize("shape", se.EXACT_SHADING_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_mlp1_bit_exact_on_new_shapes(bare, shape):
    rows = _row_counts()
    sd, x = se.exact_shading_net(shape, rows=rows[-1], device="cuda")
    bare.set_weights(1, sd)
    assert bare.net_shape(1) == tuple(shape)
    ref = se.mlp1_emulate(x, sd)
    for n in rows:
        out = bare.mlp1(x[:n])
        assert torch.equal(out, ref[:n]), f"{n} rows: " + _first_difference(out, ref[:n])


# ------------------------------------------------------------------------------------ full-frame numerics, every row
@pytest.mark.parametrize("layers,widths,skip", [((6, 6), (128, 128), "3"), ((4, 4), (256, 256), "auto"),
                                                ((8, 10), (256, 256), "auto")], ids=["6x128s3", "4x256", "10x256"])
def test_mlp_kernels_full_frame_new_shapes(layers, widths, skip, make_renderer):
    """test_mlp_kernel_exact.py's full-frame check, within the bounds it sets for the shaped nets, on shaped nets of the
    new shapes: every row of an 800x800 frame at thr 0.2, K = 8 through both kernels against the float64 emulation."""
    scene = orc.SCENE_BARBERSHOP
    sd0, sd1 = so.make_shape_weights(layers, widths, skip)
    r = make_renderer(scene, sd0, sd1)
    pose, rot = torch.tensor(scene["view_cell_center"]), torch.eye(3)
    dirs = r.generate_ray_directions(W, H)
    x0, ro, rd = r.stage0(pose, rot, dirs)
    raw0 = r.mlp0(x0)
    emu0 = me.mlp0_emulate(x0, sd0, terms=3, chunk_rows=1 << 17)
    rel0 = float((raw0.double() - emu0.double()).abs().max() / emu0.abs().max())
    s2 = r.stage2(raw0, 0.2, 8)
    x1 = r.stage3(ro, rd, s2["ray"], s2["z"])
    del x0, emu0
    raw1 = r.mlp1(x1)
    emu1 = se.mlp1_emulate(x1, sd1, chunk_rows=1 << 18)
    err = (raw1.double() - emu1.double()).abs() / emu1.double().abs().amax(0)
    max_rel, mean_rel = float(err.max()), float(err.mean())
    frac = float((err > 2.0 ** -9).any(1).double().mean())
    print(f"{layers} x {widths} skip {skip}: sampling rows {raw0.shape[0]}, shading rows {raw1.shape[0]}: split max rel "
          f"{rel0:.3e}; shading max rel {max_rel:.3e}, mean rel {mean_rel:.3e}, rows above a bf16 flip {frac:.3e}")
    b0, b1, b2, b3 = FRAME_BOUNDS["shaped"]
    assert rel0 < b0 and max_rel < b1 and mean_rel < b2 and frac < b3


# ------------------------------------------------------------------------------------------------ parity gate
def _packed_mask(g):
    return np.isfinite(g["z_nan"])


@pytest.mark.parametrize("case", list(SHAPE_CASES))
def test_shape_golden_parity_gate(case):
    """The reference's own outputs for the case's networks: identical sample counts on >= 99.9 % of the rays, PSNR >=
    49.4 dB (|dPSNR| < 0.05 dB for a 30 dB scene), and stage 2 on the reference's raw0 selects and compacts exactly the
    reference's samples."""
    g = load_golden(case)
    m = g["meta"]
    sd0, sd1 = shape_case_weights(g)
    r = _renderer(m["scene_params"], sd0, sd1)
    assert (r.net_shape(0), r.net_shape(1)) == SHAPES[case]
    out = r.render_rays(g["pose"], g["rot"], torch.from_numpy(g["dirs"]).cuda(), m["thr"], m["K"], want_oracle_weights=True)
    same = (out["n_samples"].cpu().numpy() == np.round(g["asp"] * m["K"]).astype(np.int32)).mean()
    p = orc.psnr(out["rgb"].cpu().numpy(), g["rgb"])
    print(f"{case}: identical counts {same:.4f}, PSNR(ours, reference) {p:.2f} dB")
    assert same >= 0.999 and p >= 49.4
    np.testing.assert_allclose(out["oracle_weights"].cpu().numpy(), g["raw0"], rtol=0, atol=2e-4 * max(1, np.abs(g["raw0"]).max()))
    s2 = r.stage2(torch.from_numpy(g["raw0"]).cuda(), m["thr"], m["K"])
    mask = _packed_mask(g)
    cnt = mask.sum(1)
    np.testing.assert_array_equal(s2["count"].cpu().numpy(), cnt)
    np.testing.assert_array_equal(s2["ray"].cpu().numpy(), np.nonzero(mask)[0])
    o2 = orc.stage2_sample(torch.from_numpy(g["raw0"]), m["thr"], m["K"], m["scene_params"]["depth_range"])
    np.testing.assert_array_equal(s2["cell"].cpu().numpy(), o2["cell"].numpy()[mask])
    np.testing.assert_array_equal(s2["zp"].cpu().numpy(), o2["zp"].numpy()[mask])
    r.close()


@pytest.mark.parametrize("case", list(SHAPE_CASES))
def test_shape_frame_against_oracle(case):
    """Every 16th ray of the 800 x 800 frame (40 000 rays) against the CPU oracle with the case's networks."""
    g = load_golden(case)
    m = g["meta"]
    sd0, sd1 = shape_case_weights(g)
    scene = m["scene_params"]
    dirs = torch.from_numpy(orc.generate_ray_directions(W, H, scene["fov"]).reshape(-1, 3)[::16].copy()).float()
    pose, rot = torch.from_numpy(g["pose"]), torch.from_numpy(g["rot"])
    ref_rgb, ref_n = so.render_frame(pose, rot, dirs, sd0, sd1, scene, m["thr"], m["K"])
    r = _renderer(scene, sd0, sd1)
    out = r.render_rays(pose, rot, dirs.cuda(), m["thr"], m["K"])
    rgb, n = out["rgb"].cpu(), out["n_samples"].cpu().long()
    same = (n == ref_n).float().mean().item()
    p = orc.psnr(rgb, ref_rgb)
    print(f"{case}: {dirs.shape[0]} rays, identical counts {same:.6f}, PSNR(ours, oracle) {p:.2f} dB")
    assert torch.isfinite(rgb).all() and same >= 0.999 and p >= 49.4
    r.close()


# ------------------------------------------------------------------------------------------------ modes
@pytest.mark.parametrize("shape", se.EXACT_SHADING_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_fused_encoder_equals_tiles_on_new_shapes(shape, make_renderer):
    """fuse_encoder 1 (V encoded inside the kernel after the skip consumer, or after layer 0 without a skip) renders the
    frame of fuse_encoder 0 bit for bit, and both equal the stage entry points composed by hand."""
    D, Wd, _ = shape
    sd0, sd1 = so.make_shape_weights((6, D), (128, Wd), _skip_entry(shape))
    scene = orc.SCENE_BARBERSHOP
    r = make_renderer(scene, sd0, sd1)
    assert r.net_shape(1) == tuple(shape)
    pose, rot = torch.tensor(scene["view_cell_center"]), orc.rotation_yaw(30.0)
    dirs = r.generate_ray_directions(400, 400)
    ref = _compose(r, pose, rot, dirs, 0.2, 8)
    for fuse in (0, 1):
        r.set_option("fuse_encoder", fuse)
        out = r.render_rays(pose, rot, dirs, 0.2, 8)
        assert torch.equal(out["n_samples"], ref["n_samples"]) and torch.equal(out["rgb"], ref["rgb"]), f"fuse_encoder {fuse}"
    r.set_option("fuse_encoder", 0)


def test_dense_and_sample_budget_on_a_6x128_net(make_renderer):
    sd0, sd1 = so.make_shape_weights((6, 6), (128, 128), "3")
    scene = orc.SCENE_BARBERSHOP
    r = make_renderer(scene, sd0, sd1)
    pose, rot = torch.tensor(scene["view_cell_center"]), orc.rotation_yaw(30.0)
    all_dirs = torch.from_numpy(orc.generate_ray_directions(W, H, scene["fov"]).reshape(-1, 3)).float()
    # dense K = 128 on five image rows, against the oracle.  Dense mode weights alpha by the raw sampling-net output
    # (zp = raw0), which these untrained-style nets put far outside [0, 1], so the colours are large: a relative check, as
    # test_gpu_parity.py makes for the random nets
    rows = torch.arange(5) * 160 + 37
    dirs = all_dirs[(rows[:, None] * W + torch.arange(W)[None, :]).reshape(-1)].contiguous()
    ref_rgb, ref_n = so.render_frame(pose, rot, dirs, sd0, sd1, scene, 0.0, 128, chunk=1000)
    out = r.render_rays(pose, rot, dirs.cuda(), 0.0, 128)
    rgb = out["rgb"].cpu()
    rel = float((rgb - ref_rgb).abs().max()) / max(1.0, float(ref_rgb.abs().max()))
    print(f"dense K=128, {dirs.shape[0]} rays: max |rgb| {float(ref_rgb.abs().max()):.3g}, max error / scale {rel:.3e}")
    assert torch.isfinite(rgb).all() and torch.equal(out["n_samples"].cpu().long(), ref_n) and rel < 0.05
    # a sample budget: M <= B, and the picture is that of a fixed-threshold render at the chosen threshold
    d = all_dirs.cuda()
    free = r.render_rays(pose, rot, d, 0.1, 8)
    budget = int(free["n_samples"].sum()) // 2
    r.set_option("sample_budget", budget)
    got = r.render_rays(pose, rot, d, 0.1, 8)
    t = r.last_threshold()
    r.set_option("sample_budget", 0)
    fixed = r.render_rays(pose, rot, d, t, 8)
    print(f"sample budget {budget}: threshold {t:.6g}, {int(got['n_samples'].sum())} samples")
    assert t > 0.1 and int(got["n_samples"].sum()) <= budget
    assert torch.equal(got["rgb"], fixed["rgb"]) and torch.equal(got["n_samples"], fixed["n_samples"])


# ------------------------------------------------------------------------------------------------ export path
def test_export_dir_and_viewer_render_a_6x128_net(tmp_path):
    import __graft_entry__ as g
    from adanerf_b200 import Renderer
    from adanerf_b200 import onnx_weights as ow
    scene = orc.SCENE_BARBERSHOP
    sd0, sd1 = so.make_shape_weights((6, 6), (128, 128), "3")
    d = tmp_path / "export"
    ow.write_export_dir(str(d), scene, sd0, sd1, 0.2, 8)
    r1, thr, K = Renderer.from_export_dir(str(d))
    assert (K, round(thr, 4)) == (8, 0.2)
    assert r1.net_shape(0) == (6, 128, -1) and r1.net_shape(1) == (6, 128, 3)
    r2 = _renderer(scene, sd0, sd1)
    pose, rot = torch.tensor(scene["view_cell_center"]), torch.eye(3)
    assert torch.equal(r1.render_camera(pose, rot, 200, 200, thr, K)["rgb"], r2.render_camera(pose, rot, 200, 200, 0.2, 8)["rgb"])
    r1.close()
    r2.close()
    res = subprocess.run([g.VIEWER, str(d), "-s", "400", "300", "-f", "2"], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stdout + res.stderr
    assert "net 0: sampling 6 x 128, skip -1" in res.stdout and "net 1: shading 6 x 128, skip 3" in res.stdout, res.stdout
    assert re.search(r"2 frames 400x300: ([0-9.]+) ms/frame", res.stdout), res.stdout
    assert os.path.isdir(d)


# ------------------------------------------------------------------------------------------------ rejections
def test_unsupported_shapes_are_rejected_with_the_tensor_named(bare):
    from adanerf_b200 import AdnError
    for net_id, sd, name in unsupported_nets():
        with pytest.raises(AdnError) as e:
            bare.set_weights(net_id, sd)
        assert e.value.status == 1 and name.split(" ")[0] in str(e.value), (name, str(e.value))
    with pytest.raises(AdnError) as e:   # the single pts_linears.0 tensor of test_gpu_parity.py::test_error_paths
        bare.set_weights(1, {"pts_linears.0.weight": torch.zeros(256, 60)})
    assert e.value.status == 1 and "pts_linears.0.weight" in str(e.value)
