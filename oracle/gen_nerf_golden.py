"""TEST INFRASTRUCTURE -- fixtures of the one-network branch (inFeatures = [RayMarchFromPoses], rayMarchSampler =
[LinearlySpacedZNearZFar], or [LinearlySpacedZNearZFarNoDepthRange] with useNDC: plain NeRF), written from the UNMODIFIED
reference run on CPU through oracle/ref_harness.py (build container only):

    tests/golden/nerf_<nets>_<world|ndc>_k<K>.npz    ray_d, ray_dirs, z, raw1, rgb, weights, alpha, depth_est of one
                                                     inference call, with the rays, pose and (random nets) the seed

Cases: world and NDC scenes; K in {1, 2, 64, 128}; random-init NeRF nets (oracle.adanerf_oracle.make_weights("rand"))
and the reference's shipped Pavillon shading net used as a single NeRF.  No trained NeRF export ships with the reference,
so these fixtures are the parity evidence for this branch.  The fake dataset_info gives depth_range and
depth_range_warped different values, so the fixtures pin which one the run uses (the unwarped one: no SpherePosDir).

    python oracle/gen_nerf_golden.py
"""
import math
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import ref_harness as rh          # noqa: E402
from oracle import adanerf_oracle as orc      # noqa: E402
from oracle.gen_golden import meta, save      # noqa: E402
from adanerf_b200.synthetic import load_weights_npz   # noqa: E402

CASES = [("rand", s, K) for s in ("world", "ndc") for K in (1, 2, 64, 128)] + [("pav", "world", K) for K in (64, 128)]
N_RAYS = 256


def warped_range(depth_range):
    """A depth_range_warped unlike depth_range, for the fake dataset_info: a run that used it would place other depths."""
    return [float(depth_range[0]) * 0.5, float(depth_range[1]) * 2.0]


class NerfRefRenderer(rh.RefRenderer):
    """ref_harness.RefRenderer with one network: inFeatures = [RayMarchFromPoses], rayMarchSampler =
    [LinearlySpacedZNearZFar] (NoDepthRange and normalisation None with ndc)."""

    def __init__(self, scene, K, w=800, h=800, seed=0, ndc=False):
        rh._install_stubs()
        torch.manual_seed(seed)
        from features import FeatureSet
        from models import ModelSelection
        from train_data import TrainConfig
        cfg = rh.make_config(K=K, thr=0.0, ndc=ndc)
        one = lambda v: [v[-1]]
        for key in ("inFeatures", "outFeatures", "posEnc", "posEncArgs", "raySampleInput", "multiDepthFeatures",
                    "multiDepthIgnoreValue", "multiDepthWindowSize", "activation", "layers", "layerWidth", "skips",
                    "numRaymarchSamples", "rayMarchSamplingStep", "rayMarchNormalization", "rayMarchSamplingNoise", "zNear",
                    "zFar", "losses", "lossWeights"):
            setattr(cfg, key, one(getattr(cfg, key)))
        cfg.rayMarchSampler = ["LinearlySpacedZNearZFarNoDepthRange" if ndc else "LinearlySpacedZNearZFar"]
        self.cfg = cfg
        info = rh.make_dataset_info(scene, w, h, ndc=ndc)
        info.depth_range_warped = warped_range(scene["depth_range"])
        info.use_warped_depth_range = [False]          # datasets.py:154-159 without SpherePosDir
        self.dataset_info = info
        f_in, f_out = FeatureSet.get_sets(cfg, "cpu")
        for f in list(f_in) + list(f_out):
            f.initialize(cfg, info, "cpu")
        tc = TrainConfig()
        tc.f_in, tc.f_out, tc.config_file = f_in, f_out, cfg
        tc.models = [ModelSelection.getModel(cfg, f_in[0].n_feat, 4, "cpu", 0)]
        tc.device = "cpu"
        self.tc = tc

    def load_state_dict(self, sd):
        self.tc.models[0].load_state_dict(sd, strict=True)

    def stages(self, pose, rot, dirs):
        from datasets import SampleDataWrapper, DatasetKeyConstants as D
        from features import FeatureSetKeyConstants as F
        d = {D.image_pose: pose.reshape(1, 3), D.image_rotation: rot.reshape(1, 3, 3), D.ray_directions_samples: dirs.reshape(1, -1, 3)}
        with torch.no_grad():
            outs, dicts = self.tc.inference(SampleDataWrapper([dict(d)], [], False), gradient=False, is_inference=True)
        d0 = dicts[0]
        res = dict(rgb=outs[0], z=d0[F.nerf_input_feature_z_vals], raw1=d0[F.network_output], weights=d0[F.nerf_weights_output],
                   alpha=d0[F.nerf_alpha_output], depth_est=d0[F.nerf_estimated_depth], n_outs=len(outs), keys=sorted(d0))
        return {k: (v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else v) for k, v in res.items()}


def case_inputs(nets, space, seed):
    """Scene, pose, rotation, rays and the NeRF net of one case (rays rotated here in fp64, identity rotation on both
    sides: the reference's bmm rounding depends on the host CPU)."""
    scene = dict(orc.SCENE_PAVILLON_NDC) if space == "ndc" else dict(orc.SCENE_PAVILLON if nets == "pav" else orc.SCENE_BARBERSHOP)
    if space == "ndc":
        scene["focal"] = 0.5 * scene["w"] / math.tan(0.5 * scene["fov"])
    g = torch.Generator().manual_seed(seed)
    dirs = torch.from_numpy(orc.generate_ray_directions(800, 800, scene["fov"]).reshape(-1, 3)).float()
    dirs = dirs[torch.randperm(dirs.shape[0], generator=g)[:N_RAYS]]
    pose = torch.tensor(scene["view_cell_center"]) + 0.05 * torch.randn(3, generator=g)
    rot = orc.rotation_yaw(float(seed * 13))
    dirs = (rot.double() @ dirs.double().T).T.float()
    sd = load_weights_npz(os.path.join(ROOT, "tests", "golden", "weights_pavillon"))[1] if nets == "pav" else \
        orc.make_weights("rand", seed=seed)[1]
    return scene, pose, torch.eye(3), dirs, sd


def main():
    torch.set_num_threads(8)
    for i, (nets, space, K) in enumerate(CASES):
        seed = 300 + i
        scene, pose, rot, dirs, sd = case_inputs(nets, space, seed)
        ref = NerfRefRenderer(scene, K, seed=seed, ndc=space == "ndc")
        ref.load_state_dict(sd)
        st = ref.stages(pose, rot, dirs)
        n = dirs.shape[0]
        save(f"nerf_{nets}_{space}_k{K}.npz",
             meta=meta(case=dict(nets=nets, space=space, K=K, seed=seed, n_rays=n, depth_range=list(scene["depth_range"]),
                                 depth_range_warped=warped_range(scene["depth_range"]), n_outs=st["n_outs"], keys=st["keys"]),
                       generator="oracle/gen_nerf_golden.py via oracle/ref_harness.py (unmodified reference)"),
             pose=pose.numpy(), dirs=dirs.numpy(), z=st["z"], raw1=st["raw1"].reshape(n, K, 4), rgb=st["rgb"],
             weights=st["weights"], alpha=st["alpha"], depth_est=st["depth_est"].reshape(-1))


if __name__ == "__main__":
    main()
