"""Networks of other depths, widths and skip positions than 8 x 256 / skip 4 (CPU): the oracle against the reference's
own outputs for such networks (tests/golden/shape_*, oracle/gen_shape_golden.py), the emulation's exact networks of the
new shapes, the Python export path and the C++ export loader's shape checks."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import adanerf_oracle as orc
from oracle import mlp_emulation as me
from oracle import ref_harness as rh
from oracle import shape_emulation as se
from oracle import shape_oracle as so
from adanerf_b200 import convert
from adanerf_b200 import onnx_weights as ow

SHAPE_CASES = ["shape_6x128_s3_k8_t0.2", "shape_4x256_auto_k16_t0.15", "shape_10x256_auto_k8_t0.2"]
# (layers, widths, skip) of each case, and the (D, W, skip) the library reports for its networks
SHAPES = {
    "shape_6x128_s3_k8_t0.2": ((6, 128, -1), (6, 128, 3)),
    "shape_4x256_auto_k16_t0.15": ((4, 256, -1), (4, 256, -1)),
    "shape_10x256_auto_k8_t0.2": ((8, 256, -1), (10, 256, 4)),
}


def shape_case_weights(g):
    return so.make_shape_weights(**g["meta"]["weights"])


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    from adanerf_b200 import load_library
    return load_library()


# ------------------------------------------------------------------------------------------------ oracle vs reference
@pytest.mark.parametrize("case", SHAPE_CASES)
def test_oracle_matches_shape_golden(case):
    g = load_golden(case)
    m = g["meta"]
    sd0, sd1 = shape_case_weights(g)
    assert ow.net_shapes(sd0, sd1) == SHAPES[case]
    assert so.shading_shape(sd1) == SHAPES[case][1]
    o = so.render_rays(torch.from_numpy(g["pose"]), torch.from_numpy(g["rot"]), torch.from_numpy(g["dirs"]), sd0, sd1,
                       m["scene_params"], m["thr"], m["K"])
    np.testing.assert_allclose(o["raw0"].numpy(), g["raw0"], rtol=0, atol=5e-4)
    # the reference's raw0: selection and compaction bit for bit
    s2 = orc.stage2_sample(torch.from_numpy(g["raw0"]), m["thr"], m["K"], m["scene_params"]["depth_range"])
    z = s2["z"].numpy().copy()
    z[~np.isfinite(z)] = np.nan
    np.testing.assert_array_equal(z, g["z_nan"])
    cnt = s2["count"].numpy()
    assert cnt.min() >= 1 and cnt.max() == m["K"] and len(np.unique(cnt)) > 3   # ragged 1..K samples per ray
    same = o["asp"].numpy() == g["asp"]
    assert same.mean() > 0.98
    assert np.abs(o["rgb"].numpy() - g["rgb"])[same].max() < 2e-3
    assert orc.psnr(o["rgb"].numpy()[same], g["rgb"][same]) > 60.0
    np.testing.assert_allclose(o["weights"].numpy()[same], g["weights"][same], rtol=0, atol=2e-3)


def test_make_shape_weights_defaults_equal_shaped():
    a0, a1 = so.make_shape_weights()
    b0, b1 = orc.make_weights("shaped", seed=0)
    assert list(a0) == list(b0) and list(a1) == list(b1)
    assert all(torch.equal(a0[k], b0[k]) for k in a0) and all(torch.equal(a1[k], b1[k]) for k in a1)


@pytest.mark.skipif(not rh.available(), reason="needs the reference sources")
@pytest.mark.parametrize("layers,widths,skips,expect", [
    ((6, 6), (128, 128), ("", "3"), ((6, 128, -1), (6, 128, 3))),
    ((4, 4), (256, 256), ("", "auto"), ((4, 256, -1), (4, 256, -1))),
    ((8, 10), (256, 256), ("", "auto"), ((8, 256, -1), (10, 256, 4))),
])
def test_reference_models_have_the_inferred_shapes(layers, widths, skips, expect):
    """The reference builds its models from layers / layerWidth / skips (ModelSelection.getModel); the shape read back
    from their state_dicts is the one asked for, and the adapter takes the models as they are."""
    from adanerf_b200.adapter import B200Inference
    r = so.RefRenderer(orc.SCENE_BARBERSHOP, layers=layers, layerWidth=widths, skips=skips)
    r.tc.dataset_info = r.dataset_info   # set by TrainConfig.initialize
    scene, models, thr, K = B200Inference.args_from_train_config(r.tc)
    sd0, sd1 = models[0].state_dict(), models[1].state_dict()
    assert convert.check_state_dicts(sd0, sd1) == expect
    assert (K, thr) == (8, pytest.approx(0.2))


# ------------------------------------------------------------------------------------------------ emulation
@pytest.mark.parametrize("terms", [3, 1])
@pytest.mark.parametrize("shape", se.EXACT_SAMPLING_SHAPES_W128, ids=lambda s: "x".join(map(str, s)))
def test_exact_sampling_nets_w128_pass_their_self_check(shape, terms):
    n_in, depth, n_out, width = shape
    sd, x = se.exact_sampling_net(n_in, depth, n_out, terms, rows=1024, width=width)
    assert sd["layers.0.weight"].shape == (width if depth > 1 else n_out, n_in)
    me.check_sampling_exact(sd, x, terms)
    again, x2 = se.exact_sampling_net(n_in, depth, n_out, terms, rows=700, width=width)
    assert all(torch.equal(sd[k], again[k]) for k in sd) and torch.equal(x[:700], x2)


@pytest.mark.parametrize("shape", se.EXACT_SHADING_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_exact_shading_nets_of_new_shapes_pass_their_self_check(shape):
    sd, x = se.exact_shading_net(shape, rows=1024)
    assert so.shading_shape(sd) == tuple(shape)
    reach = se.check_shading_exact(sd, x)
    assert f"pts_linears.{shape[0] - 1}.weight" in reach and "views_linears.0.weight" in reach


def test_shape_modules_restate_the_default_net_exactly():
    """On the default 8 x 256 / skip 4 net the shape-general oracle and emulation compute what adanerf_oracle and
    mlp_emulation compute, bit for bit."""
    sd, x = me.exact_shading_net()
    assert so.shading_shape(sd) == se.DEFAULT_SHADING_SHAPE
    assert torch.equal(se.mlp1_emulate(x, sd), me.mlp1_emulate(x, sd))
    se.check_shading_exact(sd, x)
    _, sd1 = orc.make_weights("shaped", seed=0)
    x1 = torch.rand(300, 90, generator=torch.Generator().manual_seed(3)) * 2 - 1
    assert torch.equal(so.mlp1_forward(x1, sd1), orc.mlp1_forward(x1, sd1))
    sd0, _ = orc.make_weights("shaped", seed=0)
    scene, pose = orc.SCENE_BARBERSHOP, torch.tensor(orc.SCENE_BARBERSHOP["view_cell_center"])
    dirs = torch.from_numpy(orc.generate_ray_directions(64, 48, scene["fov"]).reshape(-1, 3)).float()
    for thr, K in ((0.2, 8), (0.0, 128)):
        a = so.render_rays(pose, orc.rotation_yaw(30.0), dirs, sd0, sd1, scene, thr, K)
        b = orc.render_rays(pose, orc.rotation_yaw(30.0), dirs, sd0, sd1, scene, thr, K)
        assert torch.equal(a["rgb"], b["rgb"]) and torch.equal(a["n_samples"], b["n_samples"])


@pytest.mark.parametrize("layers,widths,skip", [((6, 6), (128, 128), "3"), ((4, 4), (256, 256), "auto"),
                                                ((8, 10), (256, 256), "auto"), ((6, 8), (128, 128), "auto")])
def test_emulation_matches_oracle_on_shaped_nets(layers, widths, skip):
    """The emulation runs the same networks as the oracle: within bf16 / split rounding of mlp0_forward / mlp1_forward."""
    sd0, sd1 = so.make_shape_weights(layers, widths, skip)
    g = torch.Generator().manual_seed(5)
    x0 = torch.rand(512, 90, generator=g) * 2 - 1
    ref0 = orc.mlp0_forward(x0.double(), orc.to_dtype(sd0, torch.float64))
    assert float((me.mlp0_emulate(x0, sd0, terms=3).double() - ref0).abs().max() / ref0.abs().max()) < 2.0 ** -14
    x1 = torch.rand(512, 90, generator=g) * 2 - 1
    ref1 = so.mlp1_forward(x1.double(), orc.to_dtype(sd1, torch.float64))
    assert float((se.mlp1_emulate(x1, sd1).double() - ref1).abs().max() / ref1.abs().max()) < 2.0 ** -5


# ------------------------------------------------------------------------------------------------ export path
def _export_6x128(tmp_path):
    sd0, sd1 = so.make_shape_weights((6, 6), (128, 128), "3")
    torch.save(sd0, tmp_path / "Net0_opt.weights")
    torch.save(sd1, tmp_path / "Net1_opt.weights")
    scene = orc.SCENE_BARBERSHOP
    with open(tmp_path / "dataset_info.txt", "w") as f:
        for k in ("view_cell_center", "view_cell_size", "depth_range", "fov", "max_depth"):
            f.write(f"{k} = {scene[k]}\n")
    out = tmp_path / "export"
    convert.main(["--weights0", str(tmp_path / "Net0_opt.weights"), "--weights1", str(tmp_path / "Net1_opt.weights"),
                  "--dataset-info", str(tmp_path / "dataset_info.txt"), "--threshold", "0.2", "--samples", "8", "--out", str(out)])
    return out, sd0, sd1


def test_convert_round_trips_a_6x128_export(lib, tmp_path):
    from adanerf_b200._lib import Scene
    out, sd0, sd1 = _export_6x128(tmp_path)
    cfg = (out / "config.ini").read_text()
    assert "layers = [6, 6]" in cfg and "layerWidth = [128, 128]" in cfg and "skips = [, 3]" in cfg
    for i, sd in enumerate((sd0, sd1)):
        back = ow.read_onnx_initializers(str(out / f"model{i}.onnx"))
        assert list(back) == list(sd)
        for k, v in sd.items():
            np.testing.assert_array_equal(back[k], v.numpy())
    sc, thr, K, nt = Scene(), C.c_float(), C.c_int(), (C.c_int * 2)()
    assert lib.adn_probe_export_dir(str(out).encode(), C.byref(sc), C.byref(thr), C.byref(K), nt) == 0
    assert K.value == 8 and list(nt) == [len(sd0), len(sd1)]


@pytest.mark.parametrize("key,value", [("layers", "[6, 8]"), ("layers", "[8, 6]"), ("layerWidth", "[128, 256]"),
                                       ("layerWidth", "[256, 128]")])
def test_config_ini_contradicting_the_onnx_shapes_is_rejected(lib, tmp_path, key, value):
    out, _, _ = _export_6x128(tmp_path)
    cfg = (out / "config.ini").read_text()
    assert lib.adn_probe_export_dir(str(out).encode(), None, None, None, None) == 0
    lines = [f"{key} = {value}" if ln.startswith(key + " =") else ln for ln in cfg.splitlines()]
    (out / "config.ini").write_text("\n".join(lines) + "\n")
    assert lib.adn_probe_export_dir(str(out).encode(), None, None, None, None) == 5   # ADN_ERR_IO
    # without the keys the shapes come from the ONNX initialisers alone
    (out / "config.ini").write_text("\n".join(ln for ln in lines if not ln.startswith(key + " =")) + "\n")
    assert lib.adn_probe_export_dir(str(out).encode(), None, None, None, None) == 0


def test_skips_entry_rebuilds_the_net_in_the_reference():
    """config.ini's skips entry: auto for the default skip and for no skip at D <= 4, else the skip, else a layer the net
    never reaches."""
    assert ow._skips_entry(8, 4) == "auto" and ow._skips_entry(4, -1) == "auto" and ow._skips_entry(10, 4) == "auto"
    assert ow._skips_entry(6, 3) == "3" and ow._skips_entry(6, -1) == "6"


def unsupported_nets():
    """(net_id, state dict, name of the offending tensor) for every kind of shape the library rejects."""
    sd0, sd1 = so.make_shape_weights((6, 6), (128, 128), "3")
    out = []
    for W in (64, 192):
        s0, s1 = orc.init_sampling_net(W=W, D=4), orc.init_shading_net(W=W, D=4)
        out.append((0, s0, "layers.0.weight"))
        out.append((1, s1, "pts_linears.0.weight"))
    # a BaseNet skip: a hidden layer that reads more than W columns
    s = dict(sd0)
    s["layers.3.weight"] = torch.zeros(128, 128 + 90)
    out.append((0, s, "layers.3.weight"))
    # widths that do not chain
    s = dict(sd0)
    s["layers.2.weight"], s["layers.2.bias"] = torch.zeros(256, 128), torch.zeros(256)
    out.append((0, s, "layers.2.weight"))
    s = dict(sd1)
    s["pts_linears.2.weight"] = torch.zeros(128, 100)
    out.append((1, s, "pts_linears.2.weight"))
    # two skips
    s = dict(sd1)
    s["pts_linears.2.weight"] = torch.zeros(128, 128 + 63)
    out.append((1, s, "pts_linears.4.weight"))
    # a shading posEnc other than 10-4: pts (2-2: 15 columns) and views (2-2: 15 + W columns)
    s = dict(sd1)
    s["pts_linears.0.weight"] = torch.zeros(128, 15)
    out.append((1, s, "pts_linears.0.weight"))
    s = dict(sd1)
    s["views_linears.0.weight"] = torch.zeros(64, 128 + 15)
    out.append((1, s, "views_linears.0.weight"))
    # too deep: 11 pts layers
    out.append((1, orc.init_shading_net(W=128, D=11, skips=(4,)), "pts_linears.0 .. 10"))
    return out


def test_check_state_dicts_rejects_what_the_library_rejects():
    sd0, sd1 = so.make_shape_weights((6, 6), (128, 128), "3")
    assert convert.check_state_dicts(sd0, sd1) == ((6, 128, -1), (6, 128, 3))
    for net_id, sd, name in unsupported_nets():
        args = (sd, sd1) if net_id == 0 else (sd0, sd)
        with pytest.raises(ValueError) as e:
            convert.check_state_dicts(*args)
        assert name.split(" ")[0] in str(e.value), (name, str(e.value))
