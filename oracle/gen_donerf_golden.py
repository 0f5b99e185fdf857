"""TEST INFRASTRUCTURE -- fixtures of the fixed-K branch (rayMarchSampler = [none, FromClassifiedDepth], DONeRF's sampler),
written from the UNMODIFIED reference run on CPU through oracle/ref_harness.py (build container only):

    tests/golden/donerf_<nets>_<transform>_k<K>.npz    raw0, z, raw1, rgb, weights, alpha, depth_est of one inference call,
                                                       with the rays, pose and (random nets) the seed that rebuilds them

Cases: sigmoid (losses[0] = BCEWithLogitsLoss) and softmax (CrossEntropyLoss); K in {1, 4, 8, 16}; random-init nets
(oracle.adanerf_oracle.make_weights("rand")) and the reference's shipped Pavillon networks used as a DONeRF pair (their
trained raw0 gives peaked distributions).  No trained DONeRF export ships with the reference, so these fixtures are the
parity evidence for this branch.

    python oracle/gen_donerf_golden.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import ref_harness as rh          # noqa: E402
from oracle import adanerf_oracle as orc      # noqa: E402
from oracle.gen_golden import meta, save      # noqa: E402
from adanerf_b200.synthetic import load_weights_npz   # noqa: E402

LOSSES = {"sigmoid": "BCEWithLogitsLoss", "softmax": "CrossEntropyLoss"}
CASES = [("rand", t, K) for t in LOSSES for K in (1, 4, 8, 16)] + [("pav", t, K) for t in LOSSES for K in (4, 16)]
N_RAYS = 384


class DonerfRefRenderer(rh.RefRenderer):
    """ref_harness.RefRenderer with rayMarchSampler = [none, FromClassifiedDepth] and losses[0] = `loss0`."""

    def __init__(self, scene, K, loss0, w=800, h=800, seed=0):
        rh._install_stubs()
        torch.manual_seed(seed)
        from features import FeatureSet
        from models import ModelSelection
        from train_data import TrainConfig
        self.cfg = rh.make_config(K=K, thr=0.0)
        self.cfg.rayMarchSampler = ["none", "FromClassifiedDepth"]
        self.cfg.losses = [loss0, "MSE"]
        self.dataset_info = rh.make_dataset_info(scene, w, h)
        f_in, f_out = FeatureSet.get_sets(self.cfg, "cpu")
        for f in list(f_in) + list(f_out):
            f.initialize(self.cfg, self.dataset_info, "cpu")
        models = [ModelSelection.getModel(self.cfg, f_in[i].n_feat, 128 if i == 0 else 4, "cpu", i) for i in range(2)]
        tc = TrainConfig()
        tc.f_in, tc.f_out, tc.models, tc.config_file = f_in, f_out, models, self.cfg
        tc.device = "cpu"
        self.tc = tc


def case_inputs(nets, seed):
    """Scene, pose, rotation, rays and networks of one case (rays rotated here in fp64, identity rotation on both sides:
    the reference's bmm rounding depends on the host CPU)."""
    scene = orc.SCENE_PAVILLON if nets == "pav" else orc.SCENE_BARBERSHOP
    g = torch.Generator().manual_seed(seed)
    dirs = torch.from_numpy(orc.generate_ray_directions(800, 800, scene["fov"]).reshape(-1, 3)).float()
    dirs = dirs[torch.randperm(dirs.shape[0], generator=g)[:N_RAYS]]
    pose = torch.tensor(scene["view_cell_center"]) + 0.05 * torch.randn(3, generator=g)
    rot = orc.rotation_yaw(float(seed * 13))
    dirs = (rot.double() @ dirs.double().T).T.float()
    if nets == "pav":
        sd0, sd1 = load_weights_npz(os.path.join(ROOT, "tests", "golden", "weights_pavillon"))
    else:
        sd0, sd1 = orc.make_weights("rand", seed=seed)
    return scene, pose, torch.eye(3), dirs, sd0, sd1


def main():
    torch.set_num_threads(8)
    for i, (nets, tname, K) in enumerate(CASES):
        seed = 100 + i
        scene, pose, rot, dirs, sd0, sd1 = case_inputs(nets, seed)
        ref = DonerfRefRenderer(scene, K, LOSSES[tname], seed=seed)
        ref.load_state_dicts(sd0, sd1)
        st = ref.stages(pose, rot, dirs)
        n = dirs.shape[0]
        save(f"donerf_{nets}_{tname}_k{K}.npz",
             meta=meta(case=dict(nets=nets, transform=tname, loss0=LOSSES[tname], K=K, seed=seed, n_rays=n),
                       generator="oracle/gen_donerf_golden.py via oracle/ref_harness.py (unmodified reference)"),
             pose=pose.numpy(), dirs=dirs.numpy(), raw0=st["raw0"], ray_d=st["ray_d"], z=st["z"],
             raw1=st["raw1"].reshape(n, K, 4), rgb=st["rgb"], weights=st["weights"], alpha=st["alpha"],
             depth_est=st["depth_est"].reshape(-1))


if __name__ == "__main__":
    main()
