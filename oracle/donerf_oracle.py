"""CPU ORACLE -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The fixed-K branch of the reference (rayMarchSampler = [none, FromClassifiedDepth], the DONeRF sampler that AdaNeRF is
measured against), restated on torch-CPU tensors next to oracle/adanerf_oracle.py, whose stages 0, 1, 3 and 4 it reuses:

    rays -> SpherePosDir features -> sampling MLP -> transform + inverse-CDF placement of K samples
         -> positional encoding -> shading MLP -> density composite (nerf_raw2outputs)

Every function cites the reference lines (relative to the reference checkout) it restates.  Pinned against the live
reference by oracle/gen_donerf_golden.py (tests/golden/donerf_*.npz) and tests/test_donerf_oracle.py.

FromClassifiedDepth returns z only, so RayMarchFromPoses passes no OracleWeights to nerf_raw2outputs when losses[0] is
one of the transform losses (features.py:503-504, 563-566): accumulationMult does not reach this branch.
"""
import torch

from oracle import adanerf_oracle as orc

# losses[0] -> the transform FromClassifiedDepth.__init__ applies to raw0 (src/nerf_raymarch_common.py:625-637)
SIGMOID, SOFTMAX = 1, 2
LOSS_TRANSFORM = {"BCEWithLogitsLoss": SIGMOID, "CrossEntropyLoss": SOFTMAX, "CrossEntropyLossWeighted": SOFTMAX}


def sample_pdf(bins, weights, n_samples):
    """nerf_sample_pdf(bins, weights, n_samples, det=True) -- src/nerf_raymarch_common.py:160-192, same operation order."""
    weights = weights + 1e-5                                               # :162
    pdf = weights / torch.sum(weights, -1, keepdim=True)                   # :163
    cdf = torch.cumsum(pdf, -1)                                            # :164
    cdf = torch.cat([torch.zeros_like(cdf[..., :1]), cdf], -1)             # :165
    u = torch.linspace(0., 1., steps=n_samples, dtype=weights.dtype)       # :169-170
    u = u.expand(list(cdf.shape[:-1]) + [n_samples]).contiguous()
    inds = torch.searchsorted(cdf, u, right=True)                          # :177
    below = torch.max(torch.zeros_like(inds - 1), inds - 1)                # :178
    above = torch.min((cdf.shape[-1] - 1) * torch.ones_like(inds), inds)   # :179
    inds_g = torch.stack([below, above], -1)
    matched_shape = [inds_g.shape[0], inds_g.shape[1], cdf.shape[-1]]
    cdf_g = torch.gather(cdf.unsqueeze(1).expand(matched_shape), 2, inds_g)     # :185-186
    bins_g = torch.gather(bins.unsqueeze(1).expand(matched_shape), 2, inds_g)
    denom = cdf_g[..., 1] - cdf_g[..., 0]                                  # :188
    denom = torch.where(denom < 1e-5, torch.ones_like(denom), denom)       # :189
    t = (u - cdf_g[..., 0]) / denom                                        # :190
    return bins_g[..., 0] + t * (bins_g[..., 1] - bins_g[..., 0])          # :191


def pdf_sample(raw0, K, transform, depth_range):
    """FromClassifiedDepth.generate -- src/nerf_raymarch_common.py:642-657: raw0 [N,128] -> world z [N,K] (ascending)."""
    depth = raw0
    if transform == SIGMOID:                                               # :630-631
        depth = torch.sigmoid(depth)
    elif transform == SOFTMAX:                                             # :632-635 (softmaxselect over disc = 128: the same)
        depth = torch.nn.functional.softmax(depth, dim=-1)
    else:
        raise ValueError("transform must be SIGMOID or SOFTMAX")
    mids = torch.linspace(0., 1., depth.shape[-1] + 1, dtype=torch.float32).repeat(depth.shape[0], 1)   # :651-652
    z = sample_pdf(mids, depth, K + 2)[:, 1:-1]                            # :654-655
    return orc.log_to_world(z, depth_range)                                # :657


def nerf_raw2outputs(raw, z_vals, rays_d):
    """src/nerf_raymarch_common.py:19-68 without noise, white background or OracleWeights: raw [N,K,4], z_vals [N,K],
    rays_d [N,3] -> dict(rgb, disp, acc, weights, depth_map, alpha)."""
    dists = z_vals[..., 1:] - z_vals[..., :-1]                             # :35
    dists = torch.cat([dists, (torch.ones(1, dtype=raw.dtype) * 1e10).expand(dists[..., :1].shape)], -1)   # :36-37
    dists = dists * torch.norm(rays_d[..., None, :], dim=-1)               # :39
    rgb = torch.sigmoid(raw[..., :3])                                      # :41
    alpha = 1. - torch.exp(-torch.nn.functional.relu(raw[..., 3]) * dists)  # :33,46
    weights = alpha * torch.cumprod(torch.cat([torch.ones((alpha.shape[0], 1), dtype=raw.dtype), 1. - alpha + 1e-10], -1),
                                    -1)[:, :-1]                            # :52
    rgb_map = torch.sum(weights[..., None] * rgb, -2)                      # :58
    depth_map = torch.sum(weights * z_vals, -1)                            # :60
    disp_map = 1. / torch.max(1e-10 * torch.ones_like(depth_map), depth_map / torch.sum(weights, -1))   # :61
    acc_map = torch.sum(weights, -1)                                       # :62
    return dict(rgb=rgb_map, disp=disp_map, acc=acc_map, weights=weights, depth_map=depth_map, alpha=alpha)


def render_rays(pose, rot, dirs, sd0, sd1, scene, K, transform, return_stages=False):
    """One TrainConfig.inference call (src/train_data.py:278-299) of a FromClassifiedDepth run on one batch of rays."""
    with torch.no_grad():
        x0, ray_o, ray_d = orc.stage0_sphere_pos_dir(pose, rot, dirs, scene)
        raw0 = orc.mlp0_forward(x0, sd0)
        z = pdf_sample(raw0, K, transform, scene["depth_range"])
        x1, _, zs = orc.stage3_encode(ray_o, ray_d, z, scene, compact=False)   # features.py:458-479, every slot live
        raw1 = orc.mlp1_forward(x1, sd1)
        n = dirs.shape[0]
        comp = nerf_raw2outputs(raw1.reshape(n, K, 4), z, ray_d)           # features.py:563-566
    out = dict(rgb=comp["rgb"], n_samples=torch.full((n,), K, dtype=torch.int64))
    if return_stages:
        out.update(x0=x0, ray_o=ray_o, ray_d=ray_d, raw0=raw0, z=z, x1=x1, raw1=raw1, weights=comp["weights"],
                   alpha=comp["alpha"], depth_map=comp["depth_map"], acc=comp["acc"], disp=comp["disp"],
                   depth_est=orc.log_from_world(comp["depth_map"], scene["depth_range"]))   # features.py:576-577
    return out
