"""TEST INFRASTRUCTURE -- stores what the tests that once read the reference at run time compare against, so that they run
from the repository alone.  Runs the UNMODIFIED reference on CPU (oracle/ref_harness.py) and writes

    tests/golden/live_fresh_seed.npz     fresh-seed end-to-end runs (test_oracle_golden.py::test_live_reference_fresh_seed)
    tests/golden/live_train_config.json  what an initialised TrainConfig carries (test_adapter_config.py)
    tests/golden/viewer_sample/          the reference viewer's shipped sample export directory, its networks shrunk to one
                                         row per initialiser (test_export_loader.py::test_cxx_loader_reads_shipped_sample)

    python oracle/gen_live_golden.py
"""
import hashlib
import json
import os
import shutil
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import ref_harness as rh          # noqa: E402
from oracle import adanerf_oracle as orc      # noqa: E402
from oracle.gen_golden import OUT, meta, save  # noqa: E402
from adanerf_b200 import onnx_weights as ow   # noqa: E402

FRESH_SEEDS = [(11, 8, 0.2), (12, 4, 0.05), (13, 16, 0.3)]
TRAIN_CONFIGS = [(8, 0.2), (16, 0.15)]


def digest(t):
    return hashlib.sha256(np.ascontiguousarray(t.detach().cpu().numpy()).tobytes()).hexdigest()


def fresh_seed_inputs(seed):
    """Inputs of one fresh-seed case, rebuilt the same way by the test.  The rays are rotated here, in fp64 rounded once,
    and both sides get the identity rotation: the reference's bmm is a BLAS call whose rounding depends on the host CPU."""
    scene = orc.SCENE_BARBERSHOP
    g = torch.Generator().manual_seed(seed)
    dirs = torch.from_numpy(orc.generate_ray_directions(800, 800, scene["fov"]).reshape(-1, 3)).float()
    dirs = dirs[torch.randperm(dirs.shape[0], generator=g)[:512]]
    pose = torch.tensor(scene["view_cell_center"]) + 0.1 * torch.randn(3, generator=g)
    rot = orc.rotation_yaw(float(seed * 17))
    dirs = (rot.double() @ dirs.double().T).T.float()
    sd0, sd1 = orc.make_weights("rand", seed=seed)
    # shape the sampling net so counts are ragged
    sd0["layers.7.weight"] *= 0.15
    sd0["layers.7.bias"] = sd0["layers.7.bias"] * 0.15 - 0.2
    return scene, pose, torch.eye(3), dirs, sd0, sd1


def gen_fresh_seed():
    arrays = {}
    for seed, K, thr in FRESH_SEEDS:
        scene, pose, rot, dirs, sd0, sd1 = fresh_seed_inputs(seed)
        ref = rh.RefRenderer(scene, K=K, thr=thr, seed=seed)
        # the reference's own initialisation, as digests (the oracle's make_weights must reproduce it bit for bit)
        for i, m in enumerate(ref.models):
            for k, v in m.state_dict().items():
                arrays[f"{seed}/init{i}/{k}"] = np.array(digest(v))
        ref.load_state_dicts(sd0, sd1)
        st = ref.stages(pose, rot, dirs)
        for k in ("raw0", "asp", "rgb", "weights"):
            arrays[f"{seed}/{k}"] = np.asarray(st[k])
    save("live_fresh_seed.npz", meta=meta(cases=FRESH_SEEDS), **arrays)


def gen_train_config():
    out = dict(meta=json.loads(str(meta())), configs=[])
    for K, thr in TRAIN_CONFIGS:
        ref = rh.RefRenderer(orc.SCENE_PAVILLON, K=K, thr=thr)
        tc = ref.tc
        f1 = tc.f_in[1]
        view = ref.dataset_info.view
        out["configs"].append(dict(
            K=K, thr=thr,
            f_in1=dict(depth_range=[float(x) for x in f1.depth_range], max_depth=float(f1.max_depth), z_near=float(f1.z_near),
                       z_far=float(f1.z_far), z_sampler_threshold=float(f1.z_sampler.threshold),
                       n_ray_samples=int(f1.n_ray_samples), useNDC=bool(getattr(f1, "useNDC", False))),
            view=dict(view_cell_center=[float(x) for x in view.view_cell_center],
                      view_cell_size=[float(x) for x in view.view_cell_size], fov=float(view.fov)),
            state_dict_keys=[list(tc.models[0].state_dict().keys()), list(tc.models[1].state_dict().keys())]))
    with open(os.path.join(OUT, "live_train_config.json"), "w") as f:
        json.dump(out, f, indent=1)


def gen_viewer_sample():
    src = os.path.join(rh.REF_ROOT, "adanerf_real_time_viewer", "sample")
    dst = os.path.join(OUT, "viewer_sample")
    os.makedirs(dst, exist_ok=True)
    for f in ("config.ini", "dataset_info.txt"):
        shutil.copyfile(os.path.join(src, f), os.path.join(dst, f))
    for i in range(2):
        tensors = ow.read_onnx_initializers(os.path.join(src, f"model{i}.onnx"))
        ow.write_onnx_initializers(os.path.join(dst, f"model{i}.onnx"), {name: t[:1] for name, t in tensors.items()})


if __name__ == "__main__":
    assert rh.available(), "needs the reference checkout (ADANERF_REFERENCE)"
    gen_fresh_seed()
    gen_train_config()
    gen_viewer_sample()
