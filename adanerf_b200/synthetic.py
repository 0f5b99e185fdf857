"""Synthetic inputs for benchmarks and demos (no datasets / checkpoints offline): the scene constants of the
reference's shipped samples and random-init networks built in the construction order of the reference's classes
(BaseNet.__init__ src/models.py:71-80, NeRF.__init__ src/models.py:226-250, ModelSelection order: net 0 then net 1),
so a seed gives the reference's initial parameters.  Product-side helper: does not use anything under oracle/."""
import os

import torch

# adanerf_real_time_viewer/sample/dataset_info.txt (Barbershop)
SCENE_BARBERSHOP = dict(
    view_cell_center=[2.25, 7.75, 1.5], view_cell_size=[1.5, 1.5, 0.4],
    depth_range=[-0.42766728550195693, 7.07244257926941], fov=1.5271797180175781,
    max_depth=8.704841423034669)

# adanerf_real_time_viewer/sample_pavillon_16/dataset_info.txt (Pavillon; its trained networks ship with the reference)
SCENE_PAVILLON = dict(
    view_cell_center=[0.783, -3.19, 1.39], view_cell_size=[0.7, 0.7, 0.2],
    depth_range=[0.1542200982570648, 8.358194804191589], fov=1.1386263370513916,
    max_depth=8.79825210571289)


# the NDC / LLFF variant (configs/fine_training_ndc.ini) on the same geometry: the dataset's w, h feed ndc_rays (features.py:430)
SCENE_PAVILLON_NDC = dict(SCENE_PAVILLON, use_ndc=True, w=800, h=800)


def load_npz(path):
    """{name: array} of an .npz, or of a directory of .npz parts (large fixtures are stored split so that no file exceeds
    1 MB; the parts hold disjoint keys)."""
    import numpy as np
    parts = [os.path.join(path, f) for f in sorted(os.listdir(path)) if f.endswith(".npz")] if os.path.isdir(path) else [path]
    out = {}
    for p in parts:
        z = np.load(p, allow_pickle=False)
        out.update({k: z[k] for k in z.files})
    return out


def load_weights_npz(path):
    """(sampling, shading) state_dicts from an .npz (or a directory of .npz parts) with keys `sd0/<name>`, `sd1/<name>`
    (tests/golden/weights_pavillon: the initialisers of sample_pavillon_16/model{0,1}.onnx, the reference's shipped trained
    networks)."""
    z = load_npz(path)
    sd0 = {k[4:]: torch.from_numpy(v) for k, v in z.items() if k.startswith("sd0/")}
    sd1 = {k[4:]: torch.from_numpy(v) for k, v in z.items() if k.startswith("sd1/")}
    return sd0, sd1


def init_sampling_net(n_in=90, n_out=128, W=256, D=8):
    layers = [torch.nn.Linear(n_in, W)]
    for i in range(1, D):
        layers.append(torch.nn.Linear(W, W if i != D - 1 else n_out))
    for l in layers:
        torch.nn.init.kaiming_normal_(l.weight)
    sd = {}
    for i, l in enumerate(layers):
        sd[f"layers.{i}.weight"] = l.weight.detach().clone()
        sd[f"layers.{i}.bias"] = l.bias.detach().clone()
    return sd


def init_shading_net(input_ch=63, input_ch_views=27, W=256, D=8, skips=(4,)):
    pts = [torch.nn.Linear(input_ch, W)] + [
        torch.nn.Linear(W, W) if i not in skips else torch.nn.Linear(W + input_ch, W) for i in range(D - 1)]
    views = [torch.nn.Linear(input_ch_views + W, W // 2)]
    feature, alpha, rgb = torch.nn.Linear(W, W), torch.nn.Linear(W, 1), torch.nn.Linear(W // 2, 3)
    for l in pts + views:
        torch.nn.init.kaiming_normal_(l.weight)
    sd = {}
    for i, l in enumerate(pts):
        sd[f"pts_linears.{i}.weight"], sd[f"pts_linears.{i}.bias"] = l.weight.detach().clone(), l.bias.detach().clone()
    for name, l in (("views_linears.0", views[0]), ("feature_linear", feature), ("alpha_linear", alpha), ("rgb_linear", rgb)):
        sd[name + ".weight"], sd[name + ".bias"] = l.weight.detach().clone(), l.bias.detach().clone()
    return sd


def make_weights(kind="rand", seed=0, thr=0.2, target_spr=8.0, logits_fn=None):
    """'ndc': sampling net with 30 inputs (configs/fine_training_ndc.ini), last layer damped by a fixed recipe.
    'rand': the reference's default init (SURVEY 8d W-rand: raw logits saturate every ray at K).
    'shaped': same seed, the sampling net's last layer scaled by 0.15 and its bias shifted (bisection) until the mean
    number of cells >= thr on a probe batch is ~target_spr -> ragged 1..K samples per ray (SURVEY 8d W-shaped).
    logits_fn(sd0) -> [n,128] tensor of raw sampling-net outputs on the probe batch (the caller evaluates them with the
    renderer under test)."""
    torch.manual_seed(seed)
    sd0, sd1 = init_sampling_net(n_in=30 if kind == "ndc" else 90), init_shading_net()
    if kind == "rand":
        return sd0, sd1
    if kind == "ndc":   # posEncArgs "2-2" -> 30 input features; damped last layer: ragged 12..16 of K = 16 at thr 0.15
        sd0["layers.7.weight"] = sd0["layers.7.weight"] * 0.15
        sd0["layers.7.bias"] = sd0["layers.7.bias"] * 0.15 - 0.1
        return sd0, sd1
    if kind != "shaped":
        raise ValueError(kind)
    if logits_fn is None:
        raise ValueError("'shaped' weights need logits_fn to evaluate the probe batch")
    sd0["layers.7.weight"] = sd0["layers.7.weight"] * 0.15
    sd0["layers.7.bias"] = sd0["layers.7.bias"] * 0.15
    base = logits_fn(sd0).float().cpu()
    lo, hi = -4.0, 4.0
    for _ in range(40):
        mid = 0.5 * (lo + hi)
        if float(((base + mid) >= thr).sum(1).float().mean()) > target_spr:
            hi = mid
        else:
            lo = mid
    sd0["layers.7.bias"] = sd0["layers.7.bias"] + 0.5 * (lo + hi)
    return sd0, sd1
