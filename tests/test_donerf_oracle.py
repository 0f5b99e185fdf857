"""The fixed-K sampler (rayMarchSampler FromClassifiedDepth, DONeRF's): the CPU oracle against fixtures of the live
reference, against the live reference itself when its checkout is present, and the export-directory side (loader,
convert --sampler, the adapter's reading of a TrainConfig).  CPU only."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from adanerf_b200 import onnx_weights as ow
from adanerf_b200.synthetic import load_npz
from oracle import adanerf_oracle as orc
from oracle import donerf_oracle as dno
from oracle import ref_harness as rh
from oracle.gen_donerf_golden import CASES, LOSSES, DonerfRefRenderer, case_inputs

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TRANSFORM = {"sigmoid": dno.SIGMOID, "softmax": dno.SOFTMAX}


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    from adanerf_b200 import load_library
    return load_library()


def _scene(nets):
    return orc.SCENE_PAVILLON if nets == "pav" else orc.SCENE_BARBERSHOP


@pytest.mark.parametrize("i", range(len(CASES)), ids=[f"{n}-{t}-k{k}" for n, t, k in CASES])
def test_oracle_equals_golden(i):
    """Sampler, composite and the whole inference call of the oracle, bit for bit against the reference's fixture."""
    nets, tname, K = CASES[i]
    g = load_npz(os.path.join(GOLDEN, f"donerf_{nets}_{tname}_k{K}.npz"))
    scene = _scene(nets)
    z = dno.pdf_sample(torch.from_numpy(g["raw0"]), K, TRANSFORM[tname], scene["depth_range"])
    np.testing.assert_array_equal(z.numpy(), g["z"])
    assert (np.diff(g["z"], axis=1) >= 0).all()
    c = dno.nerf_raw2outputs(torch.from_numpy(g["raw1"]), torch.from_numpy(g["z"]), torch.from_numpy(g["ray_d"]))
    for k in ("rgb", "weights", "alpha"):
        np.testing.assert_array_equal(c[k].numpy(), g[k], err_msg=k)
    sc, pose, rot, dirs, sd0, sd1 = case_inputs(nets, 100 + i)
    np.testing.assert_array_equal(dirs.numpy(), g["dirs"])
    o = dno.render_rays(pose, rot, dirs, sd0, sd1, sc, K, TRANSFORM[tname], return_stages=True)
    for k in ("raw0", "z", "rgb", "weights", "alpha", "depth_est"):
        np.testing.assert_array_equal(o[k].numpy(), g[k], err_msg=k)
    assert (o["n_samples"] == K).all()


@pytest.mark.skipif(not rh.available(), reason="needs the reference checkout")
@pytest.mark.parametrize("seed,tname,K", [(201, "sigmoid", 8), (202, "softmax", 12), (203, "sigmoid", 3)])
def test_oracle_equals_live_reference_fresh_seed(seed, tname, K):
    """The reference's TrainConfig.inference with rayMarchSampler FromClassifiedDepth on seeds no fixture used."""
    sc, pose, rot, dirs, sd0, sd1 = case_inputs("rand", seed)
    ref = DonerfRefRenderer(sc, K, LOSSES[tname], seed=seed)
    ref.load_state_dicts(sd0, sd1)
    st = ref.stages(pose, rot, dirs)
    o = dno.render_rays(pose, rot, dirs, sd0, sd1, sc, K, TRANSFORM[tname], return_stages=True)
    np.testing.assert_array_equal(o["z"].numpy(), st["z"])
    np.testing.assert_array_equal(o["rgb"].numpy(), st["rgb"])
    np.testing.assert_array_equal(o["weights"].numpy(), st["weights"])
    np.testing.assert_array_equal(o["depth_est"].numpy(), st["depth_est"].reshape(-1))
    # the sampler returns z only: no OracleWeights reach nerf_raw2outputs, so accumulationMult has nothing to scale
    _, dicts = ref.inference(pose, rot, dirs)
    assert "OracleWeights" not in dicts[1] and "AdaptiveSamplePositions" not in dicts[1]


def test_pdf_transform_none_is_refused_by_the_oracle():
    with pytest.raises(ValueError):
        dno.pdf_sample(torch.zeros(2, 128), 4, 0, orc.SCENE_PAVILLON["depth_range"])


@pytest.mark.parametrize("loss0,transform", [("BCEWithLogitsLoss", 1), ("CrossEntropyLoss", 2), ("CrossEntropyLossWeighted", 2)])
def test_loader_accepts_donerf_export(lib, tmp_path, loss0, transform):
    sd0, sd1 = orc.make_weights("rand", seed=3)
    d = tmp_path / "export"
    ow.write_export_dir(str(d), orc.SCENE_PAVILLON, sd0, sd1, 0.0, 8, sampler="FromClassifiedDepth", sampling_loss=loss0)
    k = C.c_int()
    assert lib.adn_probe_export_dir(str(d).encode(), None, None, C.byref(k), None) == 0 and k.value == 8
    assert ow.export_sampler(str(d)) == (1, transform)


def test_loader_refuses_unsupported_samplers(lib, tmp_path, capfd):
    sd0, sd1 = orc.make_weights("rand", seed=3)
    d = tmp_path / "export"
    ow.write_export_dir(str(d), orc.SCENE_PAVILLON, sd0, sd1, 0.0, 8, sampler="FromClassifiedDepth")
    cfg = (d / "config.ini").read_text()
    # losses[0] without a transform (pdf_transform 0)
    (d / "config.ini").write_text(cfg.replace("losses = [BCEWithLogitsLoss, MSE]", "losses = [MSE, MSE]"))
    assert lib.adn_probe_export_dir(str(d).encode(), None, None, None, None) == 5
    assert "no transform" in capfd.readouterr().err
    with pytest.raises(ValueError, match="no transform"):
        ow.export_sampler(str(d))
    # another DONeRF-era sampler
    (d / "config.ini").write_text(cfg.replace("FromClassifiedDepth]", "LinearlySpacedZNearZFar]"))
    assert lib.adn_probe_export_dir(str(d).encode(), None, None, None, None) == 5
    assert "only FromClassifiedDepthAdaptive" in capfd.readouterr().err
    # FromClassifiedDepth with a depth transform other than log
    (d / "config.ini").write_text(cfg.replace("depthTransform = log", "depthTransform = linear"))
    assert lib.adn_probe_export_dir(str(d).encode(), None, None, None, None) == 5
    assert "FromClassifiedDepth exports must use" in capfd.readouterr().err
    with pytest.raises(ValueError):
        ow.write_export_dir(str(tmp_path / "x"), orc.SCENE_PAVILLON, sd0, sd1, 0.0, 8, sampler="FromClassifiedDepth",
                            sampling_loss="MSE")


def test_convert_sampler_round_trips(lib, tmp_path):
    from adanerf_b200 import convert
    sd0, sd1 = orc.make_weights("rand", seed=5)
    torch.save(sd0, tmp_path / "Net0_opt.weights")
    torch.save(sd1, tmp_path / "Net1_opt.weights")
    scene = orc.SCENE_PAVILLON
    with open(tmp_path / "dataset_info.txt", "w") as f:
        for k in ("view_cell_center", "view_cell_size", "depth_range", "fov", "max_depth"):
            f.write(f"{k} = {scene[k]}\n")
    for loss0, transform in (("BCEWithLogitsLoss", 1), ("CrossEntropyLoss", 2)):
        out = tmp_path / f"export_{transform}"
        convert.main(["--weights0", str(tmp_path / "Net0_opt.weights"), "--weights1", str(tmp_path / "Net1_opt.weights"),
                      "--dataset-info", str(tmp_path / "dataset_info.txt"), "--threshold", "0", "--samples", "16",
                      "--out", str(out), "--sampler", "FromClassifiedDepth", "--sampling-loss", loss0])
        k = C.c_int()
        assert lib.adn_probe_export_dir(str(out).encode(), None, None, C.byref(k), None) == 0 and k.value == 16
        assert ow.export_sampler(str(out)) == (1, transform)
        assert "rayMarchSampler = [none, FromClassifiedDepth]" in (out / "config.ini").read_text()
    out = tmp_path / "export_adaptive"
    convert.main(["--weights0", str(tmp_path / "Net0_opt.weights"), "--weights1", str(tmp_path / "Net1_opt.weights"),
                  "--dataset-info", str(tmp_path / "dataset_info.txt"), "--threshold", "0.2", "--samples", "8", "--out", str(out)])
    assert ow.export_sampler(str(out)) == (0, None)


def test_abi_declares_the_fixed_k_entry_points(lib):
    from adanerf_b200._lib import SYMBOLS
    for name in ("adn_pdf_sample", "adn_stage5_density_composite"):
        assert name in SYMBOLS and getattr(lib, name) is not None


@pytest.mark.skipif(not rh.available(), reason="needs the reference checkout")
def test_adapter_reads_sampler_from_train_config():
    """B200Inference.sampler_from_train_config on a TrainConfig the reference initialised for each transform loss."""
    from adanerf_b200.adapter import B200Inference
    for loss0, transform in (("BCEWithLogitsLoss", 1), ("CrossEntropyLoss", 2), ("CrossEntropyLossWeighted", 2)):
        ref = DonerfRefRenderer(orc.SCENE_PAVILLON, 8, loss0)
        assert B200Inference.sampler_from_train_config(ref.tc) == (1, transform)
        ref.tc.dataset_info = ref.dataset_info
        scene, _, thr, k = B200Inference.args_from_train_config(ref.tc)
        assert k == 8 and thr == 0.0
    ref = rh.RefRenderer(orc.SCENE_PAVILLON, K=8, thr=0.2)
    assert B200Inference.sampler_from_train_config(ref.tc) == (0, 1)
