"""`.weights` checkpoints -> export directory.

The reference saves a network as `torch.save(self.state_dict(), f"{path}{name}_{suffix}.weights")`
(src/models.py:87-90) and loads either a state_dict or a whole module (`load_weights`, src/models.py:105-112).
`src/export.py:28-93` turns a trained run into the directory the C++ viewer takes with `-mp`
({config.ini, dataset_info.txt, model0.onnx, model1.onnx}); this module does the same from two `.weights` files
without instantiating the reference's classes, so trained checkpoints run through `adn_create_from_export_dir`,
`Renderer.from_export_dir` and `adn_viewer_headless`.

    python -m adanerf_b200.convert --weights0 Net0_opt.weights --weights1 Net1_opt.weights \
        --dataset-info dataset_info.txt --threshold 0.2 --samples 8 --out export_dir \
        [--pos-enc nerf,nerf --pos-enc-args 10-4,10-4] [--sampler FromClassifiedDepth --sampling-loss BCEWithLogitsLoss]

A plain NeRF run has one network: `--sampler LinearlySpacedZNearZFar --weights0 Net0_opt.weights` (no --weights1,
--threshold or sampling net) writes {config.ini, dataset_info.txt, model0.onnx} with one-item lists; --pos-enc /
--pos-enc-args then name that one net's encoding.

The run's posEnc / posEncArgs (sampling net, shading net) go on the command line: the sampling net's split into position
and direction bands cannot be read from the width of layers.0.
"""
import argparse
import ast
from collections import OrderedDict

import torch

from .onnx_weights import PDF_TRANSFORMS, net_shapes, write_export_dir, write_nerf_export_dir
from .renderer import enc_columns

SAMPLING_KEYS = ("layers.0.weight", "layers.0.bias")
SHADING_KEYS = ("pts_linears.0.weight", "views_linears.0.weight", "feature_linear.weight", "alpha_linear.weight",
                "rgb_linear.weight")


def load_weights_file(path, allow_pickle=False):
    """state_dict (name -> fp32 CPU tensor) of a `.weights` file.  The reference saves a plain state_dict
    (src/models.py:87-90), which torch loads without executing pickled code; a file that holds a pickled nn.Module
    (older checkpoints) is only read with `allow_pickle=True` -- unpickling runs arbitrary code from the file, so that is
    the caller's explicit decision (--allow-pickle on the command line), never a silent fallback."""
    try:
        obj = torch.load(path, map_location="cpu", weights_only=True)
    except Exception as e:
        if not allow_pickle:
            raise ValueError(f"{path}: not a plain state_dict ({type(e).__name__}); pass allow_pickle=True / --allow-pickle "
                             "to unpickle it (only for files you trust)") from e
        obj = torch.load(path, map_location="cpu", weights_only=False)
    if not isinstance(obj, (dict, OrderedDict)):
        obj = obj.state_dict()
    return OrderedDict((k, v.detach().to(torch.float32).contiguous()) for k, v in obj.items() if torch.is_tensor(v))


def parse_encoding(pos_enc=("nerf", "nerf"), pos_enc_args=("10-4", "10-4")):
    """config.ini's posEnc / posEncArgs pairs (sampling net, shading net) -> ((P0, D0), (P, D)) band counts, -1 / -1 for
    posEnc none (whatever posEncArgs says, as NoEncoding ignores it; features.py:326-339).  Raises ValueError outside the
    supported encodings: shading net at most 20-10 bands, sampling net at most 20 bands in all."""
    out = []
    for e, a in zip(pos_enc, pos_enc_args):
        if e == "none" or a == "none":
            out.append((-1, -1))
        elif e == "nerf":
            try:
                p, d = (int(x) for x in a.split("-"))
            except ValueError:
                raise ValueError(f"posEncArgs {a!r}: expected P-D band counts") from None
            out.append((p, d))
        else:
            raise ValueError(f"posEnc {e!r}: only nerf and none are supported")
    (p0, d0), (p, d) = out
    if max(p, 0) > 20 or max(d, 0) > 10 or max(p0, 0) + max(d0, 0) > 20:
        raise ValueError(f"posEncArgs {list(pos_enc_args)} is outside the supported encodings "
                         "(shading net at most 20-10 bands, sampling net at most 20 bands in all)")
    return tuple(out)


DEPTH_CELLS = (32, 64, 128, 256)   # multiDepthFeatures the renderer supports: the sampling net's output width D


def check_state_dicts(sd0, sd1, encoding=None, depth_cells=128):
    """The architecture the hot path implements: BaseNet sampling net, NeRF shading net with a view branch, in the shapes
    adn_set_weights accepts (include/adanerf_b200.h): sampling net 1-12 layers of hidden width 128 or 256, D = depth_cells
    outputs (multiDepthFeatures: 32, 64, 128 or 256), no skips; shading net 1-10 pts layers of width W = 128 or 256, at most one skip, view branch W/2.
    encoding: parse_encoding's ((P0, D0), (P, D)); the input columns must be those of that encoding.  None: posEncArgs
    [10-4, 10-4] or [2-2, 10-4].
    Returns net_shapes(sd0, sd1); raises ValueError naming the offending tensor."""
    for k in SAMPLING_KEYS:
        if k not in sd0:
            raise ValueError(f"sampling net: missing {k} (expected BaseNet layers.{{i}}.weight/bias, src/models.py:71-76)")
    for k in SHADING_KEYS:
        if k not in sd1:
            raise ValueError(f"shading net: missing {k} (expected NeRF with use_viewdirs, src/models.py:214-250)")
    if encoding is None:
        n_p, n_v = 63, 27
        if sd0["layers.0.weight"].shape[1] not in (90, 30) or sd1["pts_linears.0.weight"].shape[1] != 63:
            raise ValueError(f"layers.0.weight / pts_linears.0.weight read {sd0['layers.0.weight'].shape[1]} / "
                             f"{sd1['pts_linears.0.weight'].shape[1]} columns: posEncArgs other than [10-4, 10-4] / [2-2, 10-4] "
                             "(90 or 30 / 63+27 input features) are not supported")
        enc = "posEnc 10-4"
    else:
        (p0, d0), (p, d) = encoding
        n0, n_p, n_v = enc_columns(p0) + enc_columns(d0), enc_columns(p), enc_columns(d)
        enc = "posEnc " + ("none" if p < 0 and d < 0 else f"{max(p, 0)}-{max(d, 0)}")
        if sd0["layers.0.weight"].shape[1] != n0:
            raise ValueError(f"sampling net: layers.0.weight reads {sd0['layers.0.weight'].shape[1]} columns, expected {n0} "
                             f"for posEncArgs {max(p0, 0)}-{max(d0, 0)}")
        if sd1["pts_linears.0.weight"].shape[1] != n_p:
            raise ValueError(f"shading net: pts_linears.0.weight reads {sd1['pts_linears.0.weight'].shape[1]} columns, "
                             f"expected {n_p} for {enc}")
    shapes = net_shapes(sd0, sd1)
    (d0, w0, _), (d1, w1, _) = shapes

    def expect(sd, name, rows, cols, what):
        have = tuple(sd[name].shape) if name in sd else None
        if have != (rows, cols):
            raise ValueError(f"{what}: {name} is {list(have) if have else 'missing'}, expected [{rows}, {cols}]")

    if not 1 <= d0 <= 12:
        raise ValueError(f"sampling net: layers.0 .. layers.{d0 - 1}: {d0} layers, 1-12 are supported")
    if depth_cells not in DEPTH_CELLS:
        raise ValueError(f"depth cells (multiDepthFeatures) {depth_cells}: 32, 64, 128 or 256 are supported")
    for i in range(d0):
        n_out = depth_cells if i == d0 - 1 else w0
        if i != d0 - 1 and n_out not in (128, 256):
            raise ValueError(f"sampling net: layers.{i}.weight has {n_out} outputs; the hidden width must be 128 or 256")
        expect(sd0, f"layers.{i}.weight", n_out, sd0["layers.0.weight"].shape[1] if i == 0 else w0,
               f"sampling net (no skips; layer widths must chain, {depth_cells} outputs = the depth cells)")
    if w1 not in (128, 256):
        raise ValueError(f"shading net: pts_linears.0.weight has {w1} rows; the width W must be 128 or 256")
    if not 1 <= d1 <= 10:
        raise ValueError(f"shading net: pts_linears.0 .. pts_linears.{d1 - 1}: {d1} layers, 1-10 are supported")
    n_skips = 0
    for i in range(1, d1):
        k = int(sd1[f"pts_linears.{i}.weight"].shape[1])
        n_skips += int(k == w1 + n_p)
        if n_skips > 1:
            raise ValueError(f"shading net: pts_linears.{i}.weight reads cat[pts, h] a second time; at most one skip is supported")
        expect(sd1, f"pts_linears.{i}.weight", w1, k if k == w1 + n_p else w1, f"shading net (W = {w1}, a skip reads W + {n_p})")
    for name, rows, cols in (("feature_linear", w1, w1), ("alpha_linear", 1, w1), ("views_linears.0", w1 // 2, w1 + n_v),
                             ("rgb_linear", 3, w1 // 2)):
        expect(sd1, name + ".weight", rows, cols, f"shading net (W = {w1}, {enc})")
    return shapes


def read_dataset_info(path):
    """`key = value` lines of dataset_info.txt (src/train_data.py:180-195) -> scene dict."""
    vals = {}
    with open(path) as f:
        for line in f:
            if "=" in line:
                k, v = line.split("=", 1)
                vals[k.strip()] = ast.literal_eval(v.strip())
    need = ("view_cell_center", "view_cell_size", "depth_range", "fov", "max_depth")
    missing = [k for k in need if k not in vals]
    if missing:
        raise ValueError(f"{path}: missing {missing}")
    return {k: vals[k] for k in need}


def weights_to_export_dir(weights0, weights1, out_dir, scene, threshold, num_samples, allow_pickle=False, encoding=None,
                          sampler="FromClassifiedDepthAdaptive", sampling_loss="BCEWithLogitsLoss", depth_cells=128):
    """encoding: parse_encoding's band counts; None keeps the scene's (posEncArgs [10-4, 10-4] unless it says otherwise).
    sampler / sampling_loss: rayMarchSampler and losses[0] of the run (onnx_weights.write_export_dir).  depth_cells: the
    run's multiDepthFeatures, the sampling net's output width."""
    sd0, sd1 = load_weights_file(weights0, allow_pickle), load_weights_file(weights1, allow_pickle)
    if encoding is not None:
        (p0, d0), (p, d) = encoding
        # the sampling net's 0 means "the shading net's count" in the scene: zero bands are -1 there
        scene = dict(scene, n_freq_pos=p, n_freq_dir=d, n_freq_pos0=p0 if p0 > 0 else -1, n_freq_dir0=d0 if d0 > 0 else -1)
    check_state_dicts(sd0, sd1, encoding, depth_cells)
    write_export_dir(out_dir, scene, sd0, sd1, float(threshold), int(num_samples), sampler=sampler, sampling_loss=sampling_loss)
    return sd0, sd1


def nerf_weights_to_export_dir(weights, out_dir, scene, num_samples, allow_pickle=False, encoding=None):
    """One NeRF `.weights` file -> a one-network export directory (onnx_weights.write_nerf_export_dir).  encoding: (P, D)
    band counts of the net, None keeps the scene's."""
    sd = load_weights_file(weights, allow_pickle)
    for k in SHADING_KEYS:
        if k not in sd:
            raise ValueError(f"NeRF net: missing {k} (expected NeRF with use_viewdirs, src/models.py:214-250)")
    if encoding is not None:
        scene = dict(scene, n_freq_pos=encoding[0], n_freq_dir=encoding[1])
    n_p = enc_columns(scene.get("n_freq_pos", 10))
    if sd["pts_linears.0.weight"].shape[1] != n_p:
        raise ValueError(f"NeRF net: pts_linears.0.weight reads {sd['pts_linears.0.weight'].shape[1]} columns, expected {n_p}")
    write_nerf_export_dir(out_dir, scene, sd, int(num_samples))
    return sd


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--weights0", required=True, help="sampling net checkpoint (.weights); the NeRF net of a one-network run")
    ap.add_argument("--weights1", default=None, help="shading net checkpoint (.weights); required unless --sampler LinearlySpacedZNearZFar")
    ap.add_argument("--dataset-info", required=True, help="dataset_info.txt of the run (scene constants)")
    ap.add_argument("--threshold", type=float, default=None, help="adaptiveSamplingThreshold (two-network runs)")
    ap.add_argument("--samples", type=int, required=True, help="numRaymarchSamples of the shading net (K)")
    ap.add_argument("--out", required=True)
    ap.add_argument("--allow-pickle", action="store_true",
                    help="also read checkpoints that hold a pickled nn.Module (executes code from the file: trusted files only)")
    ap.add_argument("--pos-enc", default=None, help="posEnc of the run, sampling net then shading net: nerf,nerf (default) or none")
    ap.add_argument("--pos-enc-args", default=None, help="posEncArgs of the run, e.g. 10-4,10-4 (default) or 16-4,6-2")
    ap.add_argument("--sampler", default="FromClassifiedDepthAdaptive",
                    choices=("FromClassifiedDepthAdaptive", "FromClassifiedDepth", "LinearlySpacedZNearZFar"),
                    help="rayMarchSampler of the shading net: the adaptive sampler (default), DONeRF's fixed-K FromClassifiedDepth, "
                         "or LinearlySpacedZNearZFar for a one-network NeRF run (--weights0 only)")
    ap.add_argument("--ndc", action="store_true", help="a one-network run on an NDC scene (LinearlySpacedZNearZFarNoDepthRange)")
    ap.add_argument("--z-near", type=float, default=0.001, help="zNear of a one-network run")
    ap.add_argument("--z-far", type=float, default=1.0, help="zFar of a one-network run")
    ap.add_argument("--sampling-loss", default="BCEWithLogitsLoss", choices=tuple(PDF_TRANSFORMS),
                    help="losses[0] of a FromClassifiedDepth run: sigmoid (BCEWithLogitsLoss) or softmax (the CrossEntropy losses)")
    ap.add_argument("--depth-cells", type=int, default=128, choices=DEPTH_CELLS,
                    help="multiDepthFeatures of the run: the depth cells D the sampling net classifies (its output width)")
    a = ap.parse_args(argv)
    if a.sampler == "LinearlySpacedZNearZFar":
        enc = None
        if a.pos_enc is not None or a.pos_enc_args is not None:
            enc = parse_encoding(("nerf", a.pos_enc or "nerf"), ("10-4", a.pos_enc_args or "10-4"))[1]
        scene = dict(read_dataset_info(a.dataset_info), use_ndc=a.ndc, z_near=a.z_near, z_far=a.z_far)
        nerf_weights_to_export_dir(a.weights0, a.out, scene, a.samples, a.allow_pickle, enc)
        print(f"wrote {a.out}")
        return
    if a.weights1 is None or a.threshold is None:
        ap.error("--weights1 and --threshold are required for two-network runs")
    encoding = None
    if a.pos_enc is not None or a.pos_enc_args is not None:
        split = lambda v, d: tuple(x.strip() for x in (v or d).strip("[]").split(","))
        encoding = parse_encoding(split(a.pos_enc, "nerf,nerf"), split(a.pos_enc_args, "10-4,10-4"))
    weights_to_export_dir(a.weights0, a.weights1, a.out, read_dataset_info(a.dataset_info), a.threshold, a.samples, a.allow_pickle,
                          encoding, sampler=a.sampler, sampling_loss=a.sampling_loss, depth_cells=a.depth_cells)
    print(f"wrote {a.out}")


if __name__ == "__main__":
    main()
