"""CPU ORACLE OF OTHER NETWORK SHAPES -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

oracle/adanerf_oracle.py states the hot path for the default networks (BaseNet 8 x 256, NeRF 8 x 256 with a skip at 4).
This module states what changes when the networks have another shape -- the reference's `layers`, `layerWidth` and
`skips` (src/util/config.py:55-57, ModelSelection.getModel src/models.py:363-372) -- and reuses every other stage of
adanerf_oracle unchanged:

  * `mlp1_forward` runs NeRF.forward (src/models.py:254-277) for the D, W and skip the state dict's shapes state;
  * `render_rays` / `render_frame` are adanerf_oracle's glue with that shading net;
  * `make_shape_weights` is adanerf_oracle.make_weights' "shaped" recipe for networks of any shape;
  * `RefRenderer` builds the unmodified reference's models with a given shape (oracle/ref_harness.py).

The sampling net needs nothing new: adanerf_oracle.mlp0_forward already runs any depth and width.
Pinned by tests/golden/shape_* (oracle/gen_shape_golden.py) in tests/test_net_shapes.py.
"""
import torch

from . import adanerf_oracle as orc
from . import ref_harness as rh


def shading_shape(sd1, input_ch=63):
    """(D, W, skip) of a NeRF state dict: D pts_linears of width W; a skip after layer i when pts_linears.{i+1} reads
    W + input_ch columns (models.py:226-228), -1 when there is none."""
    D = len([k for k in sd1 if k.startswith("pts_linears.") and k.endswith(".weight")])
    W = sd1["pts_linears.0.weight"].shape[0]
    skips = [i - 1 for i in range(1, D) if sd1[f"pts_linears.{i}.weight"].shape[1] == W + input_ch]
    return D, W, (skips[0] if skips else -1)


def mlp1_forward(x1, sd1, input_ch=63):
    """NeRF.forward with use_viewdirs (src/models.py:254-277) for the shape of sd1."""
    lin = torch.nn.functional.linear
    D, _, skip = shading_shape(sd1, input_ch)
    pts, views = x1[:, :input_ch], x1[:, input_ch:]
    h = pts
    for i in range(D):
        h = torch.relu(lin(h, sd1[f"pts_linears.{i}.weight"], sd1[f"pts_linears.{i}.bias"]))
        if i == skip:
            h = torch.cat([pts, h], -1)                       # :260-261 (pts first)
    alpha = lin(h, sd1["alpha_linear.weight"], sd1["alpha_linear.bias"])
    feat = lin(h, sd1["feature_linear.weight"], sd1["feature_linear.bias"])       # no activation
    h = torch.cat([feat, views], -1)                          # :266 (feature first)
    h = torch.relu(lin(h, sd1["views_linears.0.weight"], sd1["views_linears.0.bias"]))
    rgb = lin(h, sd1["rgb_linear.weight"], sd1["rgb_linear.bias"])
    return torch.cat([rgb, alpha], -1)                        # [M,4] = [rgb, alpha]


def render_rays(pose, rot, dirs, sd0, sd1, scene, thr, K):
    """adanerf_oracle.render_rays (TrainConfig.inference, src/train_data.py:278-299) with the shading net of any shape;
    non-NDC scenes.  -> dict(rgb, n_samples, asp, raw0, z, weights)."""
    with torch.no_grad():
        x0, ray_o, ray_d = orc.stage0_sphere_pos_dir(pose, rot, dirs, scene)
        raw0 = orc.mlp0_forward(x0, sd0)
        s2 = orc.stage2_sample(raw0, thr, K, scene["depth_range"])
        n = dirs.shape[0]
        dense = thr == 0.0
        x1, mapping, zs = orc.stage3_encode(ray_o, ray_d, s2["z"], scene, compact=not dense)
        raw1 = mlp1_forward(x1, sd1)
        comp = orc.stage5_composite(raw1, zs, s2["zp"], None if dense else mapping, n, K)
        n_samples = mapping.view(n, K).sum(1)
    return dict(rgb=comp["rgb"], n_samples=n_samples, asp=n_samples / K, raw0=raw0, z=s2["z"], weights=comp["weights"])


def render_frame(pose, rot, dirs, sd0, sd1, scene, thr, K, chunk=8192):
    """Chunked full-image loop -- src/evaluate.py:216-235 with inferenceChunkSize (configs/*.ini:31)."""
    rgbs, ns = [], []
    for b0 in range(0, dirs.shape[0], chunk):
        o = render_rays(pose, rot, dirs[b0:b0 + chunk], sd0, sd1, scene, thr, K)
        rgbs.append(o["rgb"])
        ns.append(o["n_samples"])
    return torch.cat(rgbs, 0), torch.cat(ns, 0)


def _shape_sampling_output(sd0, last, thr, target_spr):
    """adanerf_oracle.make_weights' 'shaped' recipe on the sampling net's last layer `last`, in place: scale it by 0.15,
    then shift its bias so that the mean number of cells >= thr is ~target_spr of 128 on the same probe batch."""
    sd0[f"layers.{last}.weight"] = sd0[f"layers.{last}.weight"] * 0.15
    sd0[f"layers.{last}.bias"] = sd0[f"layers.{last}.bias"] * 0.15
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
        if spr > target_spr:
            hi = mid
        else:
            lo = mid
    sd0[f"layers.{last}.bias"] = sd0[f"layers.{last}.bias"] + 0.5 * (lo + hi)


def make_shape_weights(layers=(8, 8), widths=(256, 256), skip="auto", seed=0, thr=0.2, target_spr=8.0):
    """'shaped' weights of networks of any supported shape: the reference's `layers`, `layerWidth` and the shading net's
    `skips` entry ("auto" = a skip at 4, models.py:210-211; an integer string = a skip there).  The same construction
    order and RNG use as the reference's (adanerf_oracle.init_sampling_net / init_shading_net); the recipe acts on the
    sampling net's layer D-1, so the rays keep ragged 1..K samples.  The defaults give adanerf_oracle.make_weights("shaped")."""
    torch.manual_seed(seed)
    sd0 = orc.init_sampling_net(W=widths[0], D=layers[0])
    sd1 = orc.init_shading_net(W=widths[1], D=layers[1], skips=(4,) if "auto" in skip else (int(skip),))
    _shape_sampling_output(sd0, layers[0] - 1, thr, target_spr)
    return sd0, sd1


class RefRenderer(rh.RefRenderer):
    """ref_harness.RefRenderer with the networks built from `layers` / `layerWidth` / `skips` (build container only)."""

    def __init__(self, scene, K=8, thr=0.2, w=800, h=800, seed=0, layers=(8, 8), layerWidth=(256, 256), skips=("", "auto")):
        rh._install_stubs()
        torch.manual_seed(seed)
        from features import FeatureSet
        from models import ModelSelection
        from train_data import TrainConfig
        self.cfg = rh.make_config(K=K, thr=thr)
        self.cfg.layers, self.cfg.layerWidth, self.cfg.skips = list(layers), list(layerWidth), list(skips)
        self.dataset_info = rh.make_dataset_info(scene, w, h)
        f_in, f_out = FeatureSet.get_sets(self.cfg, "cpu")
        for f in list(f_in) + list(f_out):
            f.initialize(self.cfg, self.dataset_info, "cpu")
        models = [ModelSelection.getModel(self.cfg, f_in[i].n_feat, 128 if i == 0 else 4, "cpu", i) for i in range(2)]
        tc = TrainConfig()
        tc.f_in, tc.f_out, tc.models, tc.config_file = f_in, f_out, models, self.cfg
        tc.device = "cpu"
        self.tc = tc
