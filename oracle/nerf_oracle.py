"""CPU ORACLE -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The one-network branch of the reference (inFeatures = [RayMarchFromPoses], rayMarchSampler = [LinearlySpacedZNearZFar],
or [LinearlySpacedZNearZFarNoDepthRange] with useNDC: plain NeRF, the baseline every sparse-sampling method is measured
against), restated on torch-CPU tensors on top of oracle/adanerf_oracle.py's encoding and NeRF forward and
oracle/donerf_oracle.py's density composite:

    rays from the camera -> K evenly spaced depths -> positional encoding -> NeRF MLP -> density composite

Every function cites the reference lines (relative to the reference checkout) it restates.  Pinned against the live
reference by oracle/gen_nerf_golden.py (tests/golden/nerf_*.npz) and tests/test_nerf_oracle.py.

Without SpherePosDir in the run, use_warped_depth_range is False (src/datasets.py:154-159), so the depths are placed and
reported with the dataset's unwarped depth_range: `scene["depth_range"]` here is that range.
"""
import torch

from oracle import adanerf_oracle as orc
from oracle import donerf_oracle as dno


def camera_rays(pose, rot, dirs, scene):
    """RayMarchFromPoses.batch's rays (src/features.py:417-431): rays_d = nerf_get_ray_dirs (a bmm, not renormalised,
    src/nerf_raymarch_common.py:147-152) and rays_o = pose for every ray.  -> (rays_o, rays_d, ray_directions), the last the
    directions RayMarchFromPoses.postprocess hands nerf_raw2outputs: rays_d, or on NDC scenes ndc_rays' un-normalised
    direction (not the unit copy that is encoded; tests/golden/nerf_*_ndc_*.npz pin this).  The rays_o / rays_d returned
    stay the world rays: orc.stage3_encode applies ndc_rays itself."""
    n = dirs.shape[0]
    rays_d = torch.transpose(torch.bmm(rot.reshape(1, 3, 3), torch.transpose(dirs.reshape(1, n, 3), 1, 2)), 1, 2).reshape(n, 3)
    rays_o = pose.reshape(1, 3).repeat(n, 1)                                # features.py:424-427 (tile)
    ndc = orc.scene_ndc(scene)
    if ndc is None:
        return rays_o, rays_d, rays_d
    _, nd = orc.ndc_rays(ndc[0], ndc[1], ndc[2], 1., rays_o, rays_d)        # :430
    return rays_o, rays_d, nd


def linear_depths(K, scene, n=1):
    """LinearlySpacedZNearZFar(NoDepthRange).generate with det = True (src/nerf_raymarch_common.py:276-289, 310-326):
    [n, K] depths, the same on every ray; world scenes warp them with LogTransform.to_world(z, depth_range)."""
    t_vals = torch.linspace(0., 1., steps=int(K + 1))[0:-1] + (0.5 / K)
    near_vec = torch.ones((n, 1)) * scene.get("z_near", 0.001)
    far_vec = torch.ones((n, 1)) * scene.get("z_far", 1.0)
    z = near_vec * (1. - t_vals) + far_vec * t_vals
    return z if scene.get("use_ndc") else orc.log_to_world(z, scene["depth_range"])


def render_rays(pose, rot, dirs, sd, scene, K, return_stages=False):
    """One TrainConfig.inference call (src/train_data.py:278-299) of a one-network run on one batch of rays."""
    with torch.no_grad():
        n = dirs.shape[0]
        ray_o, ray_d, ray_dirs = camera_rays(pose, rot, dirs, scene)
        z = linear_depths(K, scene, n)
        x1, _, _ = orc.stage3_encode(ray_o, ray_d, z, scene, compact=False,
                                     n_freq_pos=scene.get("n_freq_pos", 10), n_freq_dir=scene.get("n_freq_dir", 4))
        raw1 = orc.mlp1_forward(x1, sd, input_ch=3 + 6 * scene.get("n_freq_pos", 10))
        comp = dno.nerf_raw2outputs(raw1.reshape(n, K, 4), z, ray_dirs)     # features.py:564-567
    out = dict(rgb=comp["rgb"], n_samples=torch.full((n,), K, dtype=torch.int64))
    if return_stages:
        out.update(ray_o=ray_o, ray_d=ray_d, ray_dirs=ray_dirs, z=z, x1=x1, raw1=raw1, weights=comp["weights"],
                   alpha=comp["alpha"], depth_map=comp["depth_map"], acc=comp["acc"], disp=comp["disp"],
                   depth_est=comp["depth_map"] if scene.get("use_ndc")
                   else orc.log_from_world(comp["depth_map"], scene["depth_range"]))   # features.py:573-577
    return out
