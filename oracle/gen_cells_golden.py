"""TEST INFRASTRUCTURE -- fixtures of networks trained with D = 32, 64 or 256 depth cells (multiDepthFeatures = [D, D]),
written from the UNMODIFIED reference run on CPU through oracle/ref_harness.py (build container only):

    tests/golden/cells_<case>.npz    pose [3], rot [3,3], dirs [N,3], the reference's raw0 [N,D], z_nan [N,K] (world depth,
                                     NaN padded), asp [N], rgb [N,3] and depth_est [N,1]

No trained D != 128 model ships with the reference, so the cases are reference-initialised nets whose sampling net has D
outputs (oracle/cells_oracle.make_weights, regenerated from the seed in the meta): the "shaped" recipe, so that rays are
ragged, at several K including K = D for D = 32 and 64; one dense case (thr = 0, K = D = 64, the "dense" recipe); one NDC
case.

    python oracle/gen_cells_golden.py
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import adanerf_oracle as orc      # noqa: E402
from oracle import cells_oracle as co         # noqa: E402
from oracle.gen_golden import meta, save      # noqa: E402

# name -> (D, K, thr, kind, scene)
CASES = {
    "d32_k8": (32, 8, 0.2, "shaped", orc.SCENE_BARBERSHOP),
    "d32_k32": (32, 32, 0.2, "shaped", orc.SCENE_BARBERSHOP),
    "d64_k16": (64, 16, 0.2, "shaped", orc.SCENE_BARBERSHOP),
    "d64_k64": (64, 64, 0.2, "shaped", orc.SCENE_PAVILLON),
    "d64_dense": (64, 64, 0.0, "dense", orc.SCENE_PAVILLON),
    "d256_k16": (256, 16, 0.2, "shaped", orc.SCENE_BARBERSHOP),
    "d256_k128": (256, 128, 0.2, "shaped", orc.SCENE_PAVILLON),
    "d64_ndc_k16": (64, 16, 0.15, "ndc", orc.SCENE_PAVILLON_NDC),
}
N_RAYS = 384


def case_inputs(name, seed):
    """(scene, pose [3], rot [3,3], dirs [N,3], sd0, sd1) of a case."""
    D, K, thr, kind, scene = CASES[name]
    scene = dict(scene)
    g = torch.Generator().manual_seed(seed)
    d = torch.from_numpy(orc.generate_ray_directions(800, 800, scene["fov"]).reshape(-1, 3)).float()
    dirs = d[torch.randperm(d.shape[0], generator=g)[:N_RAYS]].contiguous()
    pose = torch.tensor(scene["view_cell_center"], dtype=torch.float32) + 0.05 * torch.randn(3, generator=g)
    rot = orc.rotation_yaw(20.0 + seed % 90)
    sd0, sd1 = co.make_weights(D, kind, seed=seed, thr=thr if thr > 0 else 0.2)
    return scene, pose, rot, dirs, sd0, sd1


def reference_stages(name, seed):
    D, K, thr, kind, _ = CASES[name]
    scene, pose, rot, dirs, sd0, sd1 = case_inputs(name, seed)
    ref = co.ref_renderer(scene, D, K, thr, seed=seed, ndc=bool(scene.get("use_ndc")))
    ref.load_state_dicts(sd0, sd1)
    st = ref.stages(pose, rot, dirs)
    out = dict(pose=pose.numpy(), rot=rot.numpy(), dirs=dirs.numpy(), raw0=st["raw0"], rgb=st["rgb"], depth_est=st["depth_est"])
    if "z_nan" in st:
        out.update(z_nan=st["z_nan"], asp=st["asp"])
    else:
        out.update(z=st["z"])
    return out


def cells_meta(**kw):
    """gen_golden.meta (torch version, thread count) with this generator's name in place of gen_golden's."""
    m = json.loads(str(meta(**kw)))
    m["generator"] = "oracle/gen_cells_golden.py via oracle/ref_harness.py (unmodified reference)"
    return np.array(json.dumps(m))


def main():
    for i, name in enumerate(CASES):
        seed = 700 + i
        D, K, thr, kind, scene = CASES[name]
        arrays = reference_stages(name, seed)
        save(f"cells_{name}.npz",
             meta=cells_meta(case=dict(name=name, D=D, K=K, thr=thr, kind=kind, seed=seed), scene_params=dict(scene), D=D,
                             K=K, thr=thr),
             **arrays)


if __name__ == "__main__":
    main()
