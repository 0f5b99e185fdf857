"""Networks trained with D = 32, 64 or 256 depth cells (multiDepthFeatures = [D, D]) on the CPU: the oracle against the
reference's fixtures (oracle/gen_cells_golden.py) and, where the checkout is present, against the live reference on fresh
seeds; the host's depth tables for D; the export loader's acceptances and refusals of multiDepthFeatures; the writer and
convert round trip."""
import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import adanerf_oracle as orc
from oracle import cells_oracle as co
from oracle import ref_harness as rh
from oracle import stage_emulation as se
from oracle.gen_cells_golden import CASES, case_inputs, reference_stages

F32 = np.float32


def _case(name):
    g = load_golden(f"cells_{name}")
    return g, g["meta"]


def _nan_padded(z):
    z = z.numpy().copy()
    z[~np.isfinite(z)] = np.nan
    return z


@pytest.mark.parametrize("name", [n for n in CASES if CASES[n][2] > 0])
def test_stage2_bit_exact_on_reference_raw0(name):
    """The reference's own raw0 [N, D]: the oracle's counts, cells, order and z equal the reference's bit for bit."""
    g, m = _case(name)
    assert g["raw0"].shape[1] == m["D"]
    sc = m["scene_params"]
    s2 = orc.stage2_sample(torch.from_numpy(g["raw0"]), m["thr"], m["K"], sc["depth_range"], no_depth_range=bool(sc.get("use_ndc")))
    np.testing.assert_array_equal(_nan_padded(s2["z"]), g["z_nan"])
    np.testing.assert_array_equal((s2["count"].numpy() / m["K"]).astype(F32), g["asp"])
    counts = s2["count"].numpy()
    assert counts.min() >= 1 and counts.max() <= m["K"]
    if m["K"] < m["D"]:
        assert len(np.unique(counts)) > 2, "the fixture's rays should be ragged"


def test_dense_case_places_one_sample_per_cell():
    g, m = _case("d64_dense")
    assert m["K"] == m["D"] == 64 and m["thr"] == 0.0
    sc = m["scene_params"]
    s2 = orc.stage2_sample(torch.from_numpy(g["raw0"]), 0.0, 64, sc["depth_range"])
    np.testing.assert_array_equal(s2["z"].numpy(), g["z"].reshape(-1, 64))
    want = s2["z"].numpy()[0]   # torch's fp32 pow; the host table's is a double pow rounded once
    np.testing.assert_array_less(np.abs(se.zlut_dense(sc, 64).astype(np.float64) - want), 2.5 * se.ulp32(want))


@pytest.mark.parametrize("name", list(CASES))
def test_end_to_end_matches_reference(name):
    """The whole oracle from the regenerated networks: raw0 to GEMM rounding, the sample sets of nearly every ray, and
    the colours of the rays whose sample set agrees."""
    g, m = _case(name)
    scene, pose, rot, dirs, sd0, sd1 = case_inputs(name, m["case"]["seed"])
    np.testing.assert_array_equal(dirs.numpy(), g["dirs"])
    o = orc.render_rays(pose, rot, dirs, sd0, sd1, scene, m["thr"], m["K"], return_stages=True)
    np.testing.assert_allclose(o["raw0"].numpy(), g["raw0"], rtol=0, atol=5e-4)
    if m["thr"] > 0:
        same = o["asp"].numpy() == g["asp"]
        assert same.mean() > 0.98
    else:
        same = np.ones(g["rgb"].shape[0], bool)
    assert np.abs(o["rgb"].numpy() - g["rgb"])[same].max() < 2e-3
    assert orc.psnr(o["rgb"].numpy()[same], g["rgb"][same]) > 60.0


@pytest.mark.skipif(not rh.available(), reason="needs the reference checkout")
@pytest.mark.parametrize("name", ["d32_k32", "d64_k16", "d256_k128", "d64_ndc_k16", "d64_dense"])
def test_oracle_equals_live_reference_on_fresh_seeds(name):
    seed = 9100 + list(CASES).index(name)
    D, K, thr, _, _ = CASES[name]
    ref = reference_stages(name, seed)
    scene, pose, rot, dirs, sd0, sd1 = case_inputs(name, seed)
    o = orc.render_rays(pose, rot, dirs, sd0, sd1, scene, thr, K, return_stages=True)
    assert ref["raw0"].shape == (dirs.shape[0], D)
    np.testing.assert_allclose(o["raw0"].numpy(), ref["raw0"], rtol=0, atol=5e-4)
    s2 = orc.stage2_sample(torch.from_numpy(ref["raw0"]), thr, K, scene["depth_range"], no_depth_range=bool(scene.get("use_ndc")))
    if thr > 0:
        np.testing.assert_array_equal(_nan_padded(s2["z"]), ref["z_nan"])
        same = o["asp"].numpy() == ref["asp"]
        assert same.mean() > 0.98
    else:
        np.testing.assert_array_equal(s2["z"].numpy(), ref["z"].reshape(-1, K))
        same = np.ones(dirs.shape[0], bool)
    assert orc.psnr(o["rgb"].numpy()[same], ref["rgb"][same]) > 60.0


# ------------------------------------------------------------------------------------------------ depth tables
@pytest.mark.parametrize("scene", [orc.SCENE_BARBERSHOP, orc.SCENE_PAVILLON, orc.SCENE_PAVILLON_NDC], ids=["barber", "pav", "ndc"])
def test_cell_tables(scene):
    """zlut(scene, 128) is the default table; every D's table is the reference's cell centres (idx + 0.5) / D warped:
    exact on NDC scenes, elsewhere within two ulps of torch's fp32 pow (of its result, before the - 1 + depth_range[0]);
    ascending."""
    assert np.array_equal(co.zlut(scene, 128).view(np.uint32), se.zlut(scene).view(np.uint32))
    for D in co.DEPTH_CELLS:
        t = co.zlut(scene, D)
        assert t.shape == (D,) and t.dtype == F32 and np.all(np.diff(t) > 0)
        centres = (torch.arange(D, dtype=torch.float32) + 0.5) * (1.0 / D)
        want = centres if scene.get("use_ndc") else orc.log_to_world(centres, scene["depth_range"])
        if scene.get("use_ndc"):
            np.testing.assert_array_equal(t, want.numpy())
        else:
            w = want.numpy() - F32(scene["depth_range"][0]) + 1   # the pow's result, before "- 1 + depth_range[0]"
            np.testing.assert_array_less(np.abs(t.astype(np.float64) - want.numpy()), 2.5 * se.ulp32(w))


@pytest.mark.parametrize("D", [32, 64, 256])
def test_packed_layout_of_a_selection(D):
    """stage_emulation.stage2_packed turns a D-cell selection into the kernels' layout: ray-major, cells ascending,
    offsets the exclusive scan of the counts, z = the D table at the cell."""
    g = torch.Generator().manual_seed(D)
    raw0 = torch.round((torch.rand(997, D, generator=g) * 1.4 - 0.9) * 32) / 32      # ties included
    lut = co.zlut(orc.SCENE_PAVILLON, D)
    for K in sorted({1, 7, min(D, 128) // 2, min(D, 128)}):
        p = se.stage2_packed(orc.stage2_sample(raw0, 0.25, K, None, no_depth_range=True), lut)
        cnt = p["count"].astype(np.int64)
        assert cnt.min() >= 1 and cnt.max() <= K and p["total"] == cnt.sum()
        np.testing.assert_array_equal(p["offset"], np.cumsum(cnt) - cnt)
        ray = p["ray"]
        assert np.all(np.diff(ray) >= 0) and np.all(np.diff(p["cell"])[np.diff(ray) == 0] > 0)
        np.testing.assert_array_equal(p["zp"], raw0.numpy()[ray, p["cell"]])
        np.testing.assert_array_equal(p["z"], lut[p["cell"]])


# ------------------------------------------------------------------------------------------------ loader / writer
@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    from adanerf_b200 import load_library
    return load_library()


def _export(tmp_path, D, name="export"):
    from adanerf_b200 import onnx_weights as ow
    sd0, sd1 = co.make_weights(D, "rand", seed=3)
    d = tmp_path / name
    ow.write_export_dir(str(d), orc.SCENE_PAVILLON, sd0, sd1, 0.2, 16)
    return d, sd0, sd1


def _set_key(d, value):
    cfg = (d / "config.ini").read_text().splitlines()
    cfg = [l for l in cfg if not l.startswith("multiDepthFeatures")]
    if value is not None:
        cfg.append(f"multiDepthFeatures = {value}")
    (d / "config.ini").write_text("\n".join(cfg) + "\n")


@pytest.mark.parametrize("D", co.DEPTH_CELLS)
def test_writer_records_depth_cells_and_loader_accepts(lib, tmp_path, D):
    d, _, _ = _export(tmp_path, D)
    assert f"multiDepthFeatures = [{D}, {D}]\n" in (d / "config.ini").read_text()
    assert lib.adn_probe_export_dir(str(d).encode(), None, None, None, None) == 0


@pytest.mark.parametrize("value", ["[64, 128]", "[48, 48]", "[0, 0]", "[512, 512]", "[64]", "[64, 64, 64]", "[abc, abc]", "[]"])
def test_loader_refuses_bad_multi_depth_features(lib, tmp_path, value):
    d, _, _ = _export(tmp_path, 64)
    _set_key(d, value)
    assert lib.adn_probe_export_dir(str(d).encode(), None, None, None, None) == 5   # ADN_ERR_IO


def test_loader_defaults_to_128_cells(lib, tmp_path):
    d, _, _ = _export(tmp_path, 128)
    _set_key(d, None)
    assert lib.adn_probe_export_dir(str(d).encode(), None, None, None, None) == 0


def test_convert_writes_depth_cells(tmp_path):
    from adanerf_b200 import convert
    from adanerf_b200 import onnx_weights as ow
    sd0, sd1 = co.make_weights(32, "rand", seed=5)
    w0, w1 = tmp_path / "Net0.weights", tmp_path / "Net1.weights"
    torch.save(sd0, w0)
    torch.save(sd1, w1)
    info = tmp_path / "dataset_info.txt"
    sc = orc.SCENE_PAVILLON
    info.write_text(f"view_cell_center = {sc['view_cell_center']}\nview_cell_size = {sc['view_cell_size']}\n"
                    f"depth_range = {sc['depth_range']}\nfov = {sc['fov']}\nmax_depth = {sc['max_depth']}\n")
    args = ["--weights0", str(w0), "--weights1", str(w1), "--dataset-info", str(info), "--threshold", "0.2", "--samples", "8"]
    with pytest.raises(ValueError, match="32 outputs|expected \\[128"):
        convert.main(args + ["--out", str(tmp_path / "a")])                       # the default D = 128 does not fit
    convert.main(args + ["--out", str(tmp_path / "b"), "--depth-cells", "32"])
    assert "multiDepthFeatures = [32, 32]\n" in (tmp_path / "b" / "config.ini").read_text()
    back = ow.read_onnx_initializers(str(tmp_path / "b" / "model0.onnx"))
    assert back["layers.7.weight"].shape == (32, 256)
    np.testing.assert_array_equal(back["layers.7.bias"], sd0["layers.7.bias"].numpy())
