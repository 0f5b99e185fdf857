"""TEST INFRASTRUCTURE -- networks trained with another number of depth cells D than the default 128 (multiDepthFeatures
= [D, D], src/features.py:250-252, src/nerf_raymarch_common.py:674-676,722-742).

oracle/adanerf_oracle.py's restatement is already D-generic: stage2_sample reads disc = raw0.shape[1], its dense path
takes K = D samples, and render_rays passes the sampling net's output through unchanged.  This module adds what depends
on D outside it:
  * zlut(scene, D): the adaptive depth table adn_create uploads for D cells (cell_depths, api.cu), bit for bit;
  * make_weights(D, ...): reference-initialised nets whose sampling net has D outputs, its last layer damped and shifted so
    that rays are ragged (oracle.make_weights' "shaped" / "ndc" recipes at D cells);
  * ref_renderer(...): the unmodified reference's TrainConfig (oracle/ref_harness.py) with multiDepthFeatures = [D, D]
    and a D-output sampling model (build container only).
"""
import torch

from oracle import adanerf_oracle as orc
from oracle import stage_emulation as se

import numpy as np

F32 = np.float32
DEPTH_CELLS = (32, 64, 128, 256)


def zlut(scene, D):
    """cell_depths(scene, D) of api.cu: (i + 0.5) * (1 / D) in fp32 (exact for D a power of 2), then to_world as
    stage_emulation.zlut does it (pow in double, the rest in fp32; NDC scenes keep the cell centre).  [D] fp32."""
    return se._to_world((np.arange(D, dtype=F32) + F32(0.5)) * F32(1.0 / D), scene)


def make_weights(D, kind="shaped", seed=0, thr=0.2, target_spr=None):
    """(sd0, sd1) in the reference's init order (oracle.make_weights) with a D-output sampling net.
    'shaped': the last layer scaled by 0.15 and its bias shifted by bisection so that the mean number of cells >= thr is
    target_spr (default D / 16) on oracle.make_weights' probe batch.  'ndc': 30 inputs, the last layer damped by
    oracle.make_weights' fixed NDC recipe.  'dense': the last layer damped to small, mostly positive outputs, so that
    dense mode's alpha = sigmoid(a) raw0 stays a fraction.  'rand': plain init."""
    torch.manual_seed(seed)
    sd0 = orc.init_sampling_net(n_in=30 if kind == "ndc" else 90, n_out=D)
    sd1 = orc.init_shading_net()
    if kind == "rand":
        return sd0, sd1
    last = "layers.7"
    if kind == "ndc":
        sd0[last + ".weight"] = sd0[last + ".weight"] * 0.15
        sd0[last + ".bias"] = sd0[last + ".bias"] * 0.15 - 0.1
        return sd0, sd1
    if kind == "dense":   # raw0 small and mostly positive: dense mode's alpha = sigmoid(a) * raw0 stays in [0, 1)
        sd0[last + ".weight"] = sd0[last + ".weight"] * 0.02
        sd0[last + ".bias"] = sd0[last + ".bias"] * 0.02 + 0.05
        return sd0, sd1
    if kind != "shaped":
        raise ValueError(kind)
    target = D / 16.0 if target_spr is None else float(target_spr)
    sd0[last + ".weight"] = sd0[last + ".weight"] * 0.15
    sd0[last + ".bias"] = sd0[last + ".bias"] * 0.15
    scene = orc.SCENE_BARBERSHOP
    dirs = torch.from_numpy(orc.generate_ray_directions(800, 800, scene["fov"]).reshape(-1, 3)[::157]).float()
    pose = torch.tensor(scene["view_cell_center"], dtype=torch.float32)
    x0, _, _ = orc.stage0_sphere_pos_dir(pose, torch.eye(3), dirs, scene)
    with torch.no_grad():
        base = orc.mlp0_forward(x0, sd0)
    lo, hi = -4.0, 4.0
    for _ in range(40):
        mid = 0.5 * (lo + hi)
        spr = float(((base + mid) >= thr).sum(1).float().mean())
        if spr > target:
            hi = mid
        else:
            lo = mid
    sd0[last + ".bias"] = sd0[last + ".bias"] + 0.5 * (lo + hi)
    return sd0, sd1


def ref_renderer(scene, D, K, thr, seed=0, ndc=False, w=800, h=800):
    """oracle/ref_harness.RefRenderer with multiDepthFeatures = [D, D]: Raw / RawSigmoid and the sampling model take D
    outputs and FromClassifiedDepthAdaptive(NoDepthRange) places cells at (idx + 0.5) / D."""
    from oracle import ref_harness as rh
    rh._install_stubs()
    torch.manual_seed(seed)
    from features import FeatureSet
    from models import ModelSelection
    from train_data import TrainConfig
    r = rh.RefRenderer.__new__(rh.RefRenderer)
    r.cfg = rh.make_config(K=K, thr=thr, ndc=ndc)
    r.cfg.multiDepthFeatures = [D, D]
    r.dataset_info = rh.make_dataset_info(scene, w, h, ndc=ndc)
    f_in, f_out = FeatureSet.get_sets(r.cfg, "cpu")
    for f in list(f_in) + list(f_out):
        f.initialize(r.cfg, r.dataset_info, "cpu")
    models = [ModelSelection.getModel(r.cfg, f_in[i].n_feat, D if i == 0 else 4, "cpu", i) for i in range(2)]
    tc = TrainConfig()
    tc.f_in, tc.f_out, tc.models, tc.config_file = f_in, f_out, models, r.cfg
    tc.device = "cpu"
    r.tc = tc
    return r
