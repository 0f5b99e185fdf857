"""Plain NeRF (one network, rayMarchSampler LinearlySpacedZNearZFar): the CPU oracle against fixtures of the live
reference and against the live reference itself when its checkout is present, the host-side depth table and the ray
kernel's emulation, and the export-directory side (loader, convert --sampler LinearlySpacedZNearZFar, the adapter's
reading of a one-network TrainConfig).  CPU only."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from adanerf_b200 import onnx_weights as ow
from adanerf_b200.synthetic import load_npz
from oracle import adanerf_oracle as orc
from oracle import donerf_oracle as dno
from oracle import nerf_oracle as nfo
from oracle import ref_harness as rh
from oracle import nerf_emulation as nem
from oracle import stage_emulation as em
from oracle.gen_nerf_golden import CASES, NerfRefRenderer, case_inputs, warped_range

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    from adanerf_b200 import load_library
    return load_library()


def _golden(nets, space, K):
    return load_npz(os.path.join(GOLDEN, f"nerf_{nets}_{space}_k{K}.npz"))


@pytest.mark.parametrize("i", range(len(CASES)), ids=[f"{n}-{s}-k{k}" for n, s, k in CASES])
def test_oracle_equals_golden(i):
    """Depths, composite and the whole inference call of the oracle, bit for bit against the reference's fixture."""
    nets, space, K = CASES[i]
    g = _golden(nets, space, K)
    scene, pose, rot, dirs, sd = case_inputs(nets, space, 300 + i)
    np.testing.assert_array_equal(dirs.numpy(), g["dirs"])
    np.testing.assert_array_equal(nfo.linear_depths(K, scene, dirs.shape[0]).numpy(), g["z"])
    _, _, ray_dirs = nfo.camera_rays(pose, rot, dirs, scene)
    c = dno.nerf_raw2outputs(torch.from_numpy(g["raw1"]), torch.from_numpy(g["z"]), ray_dirs)
    for k in ("rgb", "weights", "alpha"):
        np.testing.assert_array_equal(c[k].numpy(), g[k], err_msg=k)
    o = nfo.render_rays(pose, rot, dirs, sd, scene, K, return_stages=True)
    for k in ("z", "rgb", "weights", "alpha", "depth_est"):
        np.testing.assert_array_equal(o[k].numpy(), g[k], err_msg=k)
    np.testing.assert_array_equal(o["raw1"].numpy().reshape(-1, K, 4), g["raw1"])
    meta = json.loads(str(g["meta"]))
    assert meta["case"]["n_outs"] == 1 and "OracleWeights" not in meta["case"]["keys"]
    assert "AdaptiveSamplePositions" not in meta["case"]["keys"] and "torch_version" in meta and "threads" in meta
    if K == 1:   # nerf_raw2outputs' dists are empty at K = 1: every ray composites to black
        assert not g["rgb"].any()


@pytest.mark.parametrize("nets,K", [("rand", 64), ("pav", 128)])
def test_fixtures_use_the_unwarped_depth_range(nets, K):
    """Without SpherePosDir the run places depth with dataset_info.depth_range, not depth_range_warped."""
    g = _golden(nets, "world", K)
    scene = case_inputs(nets, "world", 0)[0]
    warped = dict(scene, depth_range=warped_range(scene["depth_range"]))
    assert not np.array_equal(nfo.linear_depths(K, warped).numpy()[0], g["z"][0])
    np.testing.assert_array_equal(nfo.linear_depths(K, scene).numpy()[0], g["z"][0])


@pytest.mark.skipif(not rh.available(), reason="needs the reference checkout")
@pytest.mark.parametrize("seed,space,K", [(401, "world", 8), (402, "ndc", 33), (403, "world", 100)])
def test_oracle_equals_live_reference_fresh_seed(seed, space, K):
    scene, pose, rot, dirs, sd = case_inputs("rand", space, seed)
    ref = NerfRefRenderer(scene, K, seed=seed, ndc=space == "ndc")
    ref.load_state_dict(sd)
    st = ref.stages(pose, rot, dirs)
    o = nfo.render_rays(pose, rot, dirs, sd, scene, K, return_stages=True)
    for k in ("z", "rgb", "weights", "alpha"):
        np.testing.assert_array_equal(o[k].numpy(), st[k], err_msg=k)
    np.testing.assert_array_equal(o["depth_est"].numpy(), st["depth_est"].reshape(-1))


@pytest.mark.parametrize("scene", [orc.SCENE_BARBERSHOP, orc.SCENE_PAVILLON, orc.SCENE_PAVILLON_NDC], ids=["barber", "pav", "ndc"])
def test_depth_table_against_torch(scene):
    """The table adn_create builds for every K (emulated by stage_emulation.zlut_dense, ATen's linspace with the fma upper
    half) against the reference's torch depths.  NDC scenes apply no warp: equal bits.  World scenes differ only through
    the to_world pow (double in the table, torch's fp32 pow in the reference): by at most two ulps of w = base^z (one from
    the pow, one from rounding (w - 1) + depth_range[0] on either side), which can be many ulps of a depth near
    depth_range[0].  Measured: 1 ulp of w on Barbershop, 2 on Pavillon."""
    n_diff = 0
    for K in range(1, 129):
        a, b = em.zlut_dense(scene, K), nfo.linear_depths(K, scene).numpy()[0]
        if scene.get("use_ndc"):
            np.testing.assert_array_equal(a, b)
            continue
        dr0 = np.float32(scene["depth_range"][0])
        w = (a - dr0) + np.float32(1)
        assert (np.abs(a.astype(np.float64) - b) <= 2 * np.spacing(w).astype(np.float64)).all(), K
        n_diff += int((a != b).sum())
    print(f"{scene.get('use_ndc') and 'ndc' or scene['depth_range']}: {n_diff} of 8256 table entries differ from torch")


@pytest.mark.parametrize("space", ["world", "ndc"])
def test_ray_emulation_against_oracle(space):
    """nerf_emulation.camera_rays (the kernel's operations) against the reference's rays: pose equal, R d within an ulp
    (the reference's bmm), on NDC scenes ndc_rays' direction within an ulp; with the identity rotation R d is exact."""
    scene, pose, rot, dirs, _ = case_inputs("rand", space, 7)
    o, d, v = nem.camera_rays(pose.numpy(), orc.rotation_yaw(20.0).numpy(), dirs.numpy(), scene)
    ro, rd, rv = nfo.camera_rays(pose, orc.rotation_yaw(20.0), dirs, scene)
    np.testing.assert_array_equal(o, ro.numpy())
    np.testing.assert_allclose(d, rd.numpy(), rtol=0, atol=2e-7)
    np.testing.assert_allclose(v, rv.numpy(), rtol=0, atol=2.4e-7)
    o, d, v = nem.camera_rays(pose.numpy(), rot.numpy(), dirs.numpy(), scene)   # identity: R d is exact on both sides
    np.testing.assert_array_equal(d, dirs.numpy())


@pytest.mark.parametrize("space", ["world", "ndc"])
def test_loader_accepts_one_network_export(lib, tmp_path, space):
    scene = dict(orc.SCENE_PAVILLON_NDC if space == "ndc" else orc.SCENE_PAVILLON, z_near=0.01, z_far=0.9)
    sd = orc.make_weights("rand", seed=3)[1]
    d = tmp_path / "export"
    ow.write_nerf_export_dir(str(d), scene, sd, 64)
    assert not (d / "model1.onnx").exists()
    k, nt = C.c_int(), (C.c_int * 2)()
    from adanerf_b200._lib import Scene
    sc = Scene()
    assert lib.adn_probe_export_dir(str(d).encode(), C.byref(sc), None, C.byref(k), nt) == 0
    assert k.value == 64 and list(nt) == [0, len(sd)] and bool(sc.use_ndc) == (space == "ndc")
    assert abs(sc.z_near - 0.01) < 1e-7 and abs(sc.z_far - 0.9) < 1e-7
    assert ow.export_sampler(str(d)) == (2, None)


def test_loader_refuses_unsupported_one_network_variants(lib, tmp_path, capfd):
    sd = orc.make_weights("rand", seed=3)[1]
    d = tmp_path / "export"
    ow.write_nerf_export_dir(str(d), orc.SCENE_PAVILLON, sd, 16)
    cfg = (d / "config.ini").read_text()
    for old, new, msg in (("[LinearlySpacedZNearZFar]", "[FromClassifiedDepthAdaptive]", "rayMarchSampler = [LinearlySpacedZNearZFar]"),
                          ("[LinearlySpacedZNearZFar]", "[LinearlySpacedZNearZFarNoDepthRange]", "rayMarchSampler = [LinearlySpacedZNearZFar]"),
                          ("rayMarchNormalization = [InverseSqrtDistCentered]", "rayMarchNormalization = [None]", "InverseSqrtDistCentered"),
                          ("depthTransform = log", "depthTransform = linear", "depthTransform = log"),
                          ("inFeatures = [RayMarchFromPoses]", "inFeatures = [RayMarchFromCoarse]", "inFeatures = [RayMarchFromPoses]")):
        (d / "config.ini").write_text(cfg.replace(old, new))
        assert lib.adn_probe_export_dir(str(d).encode(), None, None, None, None) == 5, new
        assert msg in capfd.readouterr().err, new
    nd = tmp_path / "ndc"
    ow.write_nerf_export_dir(str(nd), orc.SCENE_PAVILLON_NDC, sd, 16)
    cfg = (nd / "config.ini").read_text()
    (nd / "config.ini").write_text(cfg.replace("[LinearlySpacedZNearZFarNoDepthRange]", "[LinearlySpacedZNearZFar]"))
    assert lib.adn_probe_export_dir(str(nd).encode(), None, None, None, None) == 5
    assert "LinearlySpacedZNearZFarNoDepthRange" in capfd.readouterr().err


def test_convert_writes_one_network_export(lib, tmp_path):
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
    k, nt = C.c_int(), (C.c_int * 2)()
    assert lib.adn_probe_export_dir(str(out).encode(), None, None, C.byref(k), nt) == 0 and k.value == 32 and nt[0] == 0
    assert "rayMarchSampler = [LinearlySpacedZNearZFar]" in (out / "config.ini").read_text()
    with pytest.raises(SystemExit):   # two-network runs still need --weights1 / --threshold
        convert.main(["--weights0", str(tmp_path / "Net0_opt.weights"), "--dataset-info", str(tmp_path / "dataset_info.txt"),
                      "--samples", "32", "--out", str(tmp_path / "x")])


def test_abi_declares_the_linear_entry_points(lib):
    from adanerf_b200._lib import SYMBOLS
    for name in ("adn_camera_rays", "adn_linear_depths"):
        assert name in SYMBOLS and getattr(lib, name) is not None


@pytest.mark.skipif(not rh.available(), reason="needs the reference checkout")
@pytest.mark.parametrize("ndc", [False, True])
def test_adapter_reads_one_network_train_config(ndc):
    """args_from_train_config on a one-net TrainConfig the reference initialised: the unwarped depth_range, [None, net]."""
    from adanerf_b200.adapter import B200Inference
    scene = dict(orc.SCENE_PAVILLON_NDC if ndc else orc.SCENE_PAVILLON)
    ref = NerfRefRenderer(scene, 16, ndc=ndc)
    ref.tc.dataset_info = ref.dataset_info
    sc, models, thr, k = B200Inference.args_from_train_config(ref.tc)
    assert k == 16 and thr == 0.0 and models[0] is None and models[1] is ref.tc.models[0]
    assert sc["depth_range"] == list(scene["depth_range"]) != warped_range(scene["depth_range"])
    assert bool(sc.get("use_ndc")) == ndc
    assert B200Inference.sampler_from_train_config(ref.tc) == (2, 1)
