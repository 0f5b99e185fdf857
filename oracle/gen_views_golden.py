"""TEST INFRASTRUCTURE -- fixtures of multi-image inference: one TrainConfig.inference call over a batch of two images
(ImagePose [2,3], ImageRotation [2,3,3], RayDirectionsSamples [2,N,3]; src/train_data.py:278-299, SpherePosDir.batch /
RayMarchFromPoses.batch, src/features.py:392-427,845-864), written from the UNMODIFIED reference run on CPU through
oracle/ref_harness.py (build container only):

    tests/golden/views_<case>.npz    poses [2,3], rots [2,3,3], dirs [2,N,3], rgb [2N,3] (outs[-1]) and, for the adaptive
                                     sampler, asp [2N] (AdaptiveSamplePositions); depth_est [2N] (NeRFOutputDepth)

Cases, the two views differing in position and rotation: the shipped Pavillon pair (adaptive, K 16), an NDC pair
(make_weights("ndc"), K 16), the Pavillon pair as a DONeRF pair (FromClassifiedDepth, sigmoid, K 8) and the Pavillon shading
net as a one-network NeRF (LinearlySpacedZNearZFar, K 32).  Torch runs on one thread: with several, ATen's CPU kernels
split a two-image batch differently from a one-image batch and the last bits of the features and colours move (SURVEY).

    python oracle/gen_views_golden.py
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import ref_harness as rh          # noqa: E402
from oracle import adanerf_oracle as orc      # noqa: E402
from oracle.gen_golden import meta, save      # noqa: E402
from oracle.gen_donerf_golden import DonerfRefRenderer   # noqa: E402
from oracle.gen_nerf_golden import NerfRefRenderer       # noqa: E402
from adanerf_b200.synthetic import load_weights_npz      # noqa: E402

# name -> (sampler, scene, K, thr)
CASES = {
    "pav_k16": (0, orc.SCENE_PAVILLON, 16, 0.2),
    "ndc_k16": (0, orc.SCENE_PAVILLON_NDC, 16, 0.15),
    "donerf_pav_k8": (1, orc.SCENE_PAVILLON, 8, 0.0),
    "nerf_pav_k32": (2, orc.SCENE_PAVILLON, 32, 0.0),
}
V, N_RAYS = 2, 256


def case_inputs(name, seed):
    """Scene, the two views (poses [2,3], rots [2,3,3], dirs [2,N,3]) and the networks (sd0 None for the NeRF) of a case."""
    sampler, scene, K, thr = CASES[name]
    scene = dict(scene)
    g = torch.Generator().manual_seed(seed)
    d = torch.from_numpy(orc.generate_ray_directions(800, 800, scene["fov"]).reshape(-1, 3)).float()
    dirs = torch.stack([d[torch.randperm(d.shape[0], generator=g)[:N_RAYS]] for _ in range(V)])
    poses = torch.stack([torch.tensor(scene["view_cell_center"]) + 0.05 * torch.randn(3, generator=g) for _ in range(V)])
    rots = torch.stack([orc.rotation_yaw(25.0 + 70.0 * v) for v in range(V)])
    if name.startswith("ndc"):
        sd0, sd1 = orc.make_weights("ndc", seed=seed)
    else:
        sd0, sd1 = load_weights_npz(os.path.join(ROOT, "tests", "golden", "weights_pavillon"))
    return scene, poses, rots, dirs, (None if sampler == 2 else sd0), sd1


def reference(name, seed):
    """The reference's TrainConfig for a case, networks loaded."""
    sampler, _, K, thr = CASES[name]
    scene, _, _, _, sd0, sd1 = case_inputs(name, seed)
    t = lambda sd: {k: torch.as_tensor(v) for k, v in sd.items()}
    if sampler == 2:
        ref = NerfRefRenderer(scene, K, seed=seed)
        ref.load_state_dict(t(sd1))
    elif sampler == 1:
        ref = DonerfRefRenderer(scene, K, "BCEWithLogitsLoss", seed=seed)
        ref.load_state_dicts(t(sd0), t(sd1))
    else:
        ref = rh.RefRenderer(scene, K=K, thr=thr, seed=seed, ndc=name.startswith("ndc"))
        ref.load_state_dicts(t(sd0), t(sd1))
    return ref


def inference(ref, poses, rots, dirs):
    """TrainConfig.inference over the images of poses [n,3], rots [n,3,3], dirs [n,N,3] -> (outs, dicts)."""
    from datasets import SampleDataWrapper, DatasetKeyConstants as D
    d = {D.image_pose: poses, D.image_rotation: rots, D.ray_directions_samples: dirs}
    with torch.no_grad():
        return ref.tc.inference(SampleDataWrapper([dict(d) for _ in ref.tc.models], [], False), gradient=False, is_inference=True)


def arrays(outs, dicts):
    from features import FeatureSetKeyConstants as F
    d = dicts[-1]
    res = dict(rgb=outs[-1].numpy(), depth_est=d[F.nerf_estimated_depth].reshape(-1).numpy())
    if F.adaptive_sample_positions in d:
        res["asp"] = d[F.adaptive_sample_positions].numpy()
    return res


def main():
    torch.set_num_threads(1)
    for i, name in enumerate(CASES):
        seed = 500 + i
        _, poses, rots, dirs, _, _ = case_inputs(name, seed)
        ref = reference(name, seed)
        res = arrays(*inference(ref, poses, rots, dirs))
        sampler, scene, K, thr = CASES[name]
        save(f"views_{name}.npz",
             meta=meta(case=dict(name=name, sampler=sampler, K=K, thr=thr, seed=seed, n_views=V, n_per_view=N_RAYS),
                       generator="oracle/gen_views_golden.py via oracle/ref_harness.py (unmodified reference)"),
             poses=poses.numpy(), rots=rots.numpy(), dirs=dirs.numpy(), **res)


if __name__ == "__main__":
    main()
