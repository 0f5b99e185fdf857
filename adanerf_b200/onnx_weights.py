"""Minimal ONNX initialiser reader (no `onnx` package needed).

Reads the fp32 initialisers of the reference's exported `model{0,1}.onnx`
(writer: /root/reference/src/export.py:81-83, torch.onnx.export of BaseNet / NeRF) by walking the
protobuf wire format directly: ModelProto.graph(7) -> GraphProto.initializer(5) -> TensorProto
{dims(1), data_type(2), float_data(4), name(8), raw_data(9)}.  The C++ twin is
adanerf_b200/csrc/onnx_reader.cpp; both return tensors keyed by the state_dict names
(`layers.0.weight`, `pts_linears.3.bias`, ...) which the exporter preserves 1:1.
"""
import struct

import numpy as np


def _varint(buf, pos):
    result = 0
    shift = 0
    while True:
        if pos >= len(buf) or shift > 63:
            raise ValueError("truncated or corrupt protobuf varint")
        b = buf[pos]
        pos += 1
        result |= (b & 0x7F) << shift
        if not (b & 0x80):
            return result, pos
        shift += 7


def _fields(buf, start, end):
    """Yield (field_number, wire_type, value_or_(start,end)) for one message."""
    pos = start
    while pos < end:
        key, pos = _varint(buf, pos)
        fn, wt = key >> 3, key & 7
        if wt == 0:
            v, pos = _varint(buf, pos)
            yield fn, wt, v
        elif wt == 1:
            if pos + 8 > end:
                raise ValueError("truncated protobuf message")
            yield fn, wt, (pos, pos + 8)
            pos += 8
        elif wt == 2:
            ln, pos = _varint(buf, pos)
            if pos + ln > end:
                raise ValueError("truncated protobuf message")
            yield fn, wt, (pos, pos + ln)
            pos += ln
        elif wt == 5:
            if pos + 4 > end:
                raise ValueError("truncated protobuf message")
            yield fn, wt, (pos, pos + 4)
            pos += 4
        else:
            raise ValueError(f"unsupported protobuf wire type {wt}")


def _tensor(buf, start, end):
    dims, name, raw, dtype, floats = [], None, None, None, []
    for fn, wt, v in _fields(buf, start, end):
        if fn == 1:
            if wt == 0:
                dims.append(v)
            else:  # packed
                p, e = v
                while p < e:
                    d, p = _varint(buf, p)
                    dims.append(d)
        elif fn == 2:
            dtype = v
        elif fn == 4:
            if wt == 5:
                floats.append(struct.unpack_from("<f", buf, v[0])[0])
            else:
                floats.extend(np.frombuffer(buf, dtype="<f4", count=(v[1] - v[0]) // 4, offset=v[0]).tolist())
        elif fn == 8:
            name = bytes(buf[v[0]:v[1]]).decode("utf-8")
        elif fn == 9:
            raw = (v[0], v[1])
    if dtype != 1:  # FLOAT
        return name, None
    if raw is not None:
        arr = np.frombuffer(buf, dtype="<f4", count=(raw[1] - raw[0]) // 4, offset=raw[0]).copy()
    else:
        arr = np.asarray(floats, dtype=np.float32)
    return name, arr.reshape(dims) if dims else arr


def read_onnx_initializers(path):
    """-> dict name -> float32 ndarray (shape as stored: weights [out,in], biases [out])."""
    with open(path, "rb") as f:
        buf = memoryview(f.read())
    out = {}
    for fn, wt, v in _fields(buf, 0, len(buf)):
        if fn == 7 and wt == 2:  # graph
            for gfn, gwt, gv in _fields(buf, v[0], v[1]):
                if gfn == 5 and gwt == 2:
                    name, arr = _tensor(buf, gv[0], gv[1])
                    if arr is not None:
                        out[name] = arr
    return out


# ---------------------------------------------------------------------------------------------
# Writer (tests / tooling): emits a ModelProto whose graph carries only fp32 initialisers with raw_data,
# i.e. the part of the reference's export (src/export.py:81-83) that the renderer consumes.
def _enc_varint(v):
    out = bytearray()
    while True:
        b = v & 0x7F
        v >>= 7
        if v:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def _field(fn, wt, payload):
    key = _enc_varint((fn << 3) | wt)
    if wt == 0:
        return key + _enc_varint(payload)
    return key + _enc_varint(len(payload)) + payload


def write_onnx_initializers(path, tensors):
    """tensors: dict name -> float32 ndarray.  Layout: ModelProto{ir_version(1)=4, graph(7)=GraphProto{initializer(5)*}}."""
    graph = b""
    for name, arr in tensors.items():
        a = np.ascontiguousarray(arr, dtype="<f4")
        t = b"".join(_field(1, 0, int(d)) for d in a.shape)
        t += _field(2, 0, 1)                         # data_type = FLOAT
        t += _field(8, 2, name.encode("utf-8"))
        t += _field(9, 2, a.tobytes())               # raw_data, little endian
        graph += _field(5, 2, t)
    model = _field(1, 0, 4) + _field(7, 2, graph)
    with open(path, "wb") as f:
        f.write(model)


def net_shapes(sd0, sd1):
    """The reference's `layers`, `layerWidth` and `skips` of the two networks, read from the tensor shapes as
    adn_set_weights reads them: depth = the number of layers.{i} / pts_linears.{i} weights, width = the rows of the first,
    and a shading-net skip after layer i when pts_linears.{i+1} reads W + P columns, P = the columns of pts_linears.0
    (-1: none).  Returns ((D0, W0, -1), (D1, W1, skip))."""
    def depth(sd, prefix):
        d = 0
        while f"{prefix}{d}.weight" in sd:
            d += 1
        return d
    return (depth(sd0, "layers."), int(sd0["layers.0.weight"].shape[0]), -1), shading_shape(sd1)


def shading_shape(sd1):
    """(D, W, skip) of a NeRF net, as net_shapes reads the shading net."""
    d1 = 0
    while f"pts_linears.{d1}.weight" in sd1:
        d1 += 1
    w1, p = int(sd1["pts_linears.0.weight"].shape[0]), int(sd1["pts_linears.0.weight"].shape[1])
    skips = [i - 1 for i in range(1, d1) if int(sd1[f"pts_linears.{i}.weight"].shape[1]) == w1 + p]
    return d1, w1, skips[0] if skips else -1


def _skips_entry(depth, skip):
    """The shading net's `skips` config entry that builds this net in the reference (models.py:210-213): "auto" is a skip
    at 4 for D >= 6 and none for D <= 4; otherwise the skip layer, or for no skip a layer index the net never reaches."""
    if skip == 4 or (skip < 0 and depth <= 4):
        return "auto"
    return str(skip if skip >= 0 else depth)


def _enc_entries(scene):
    """config.ini's posEnc and posEncArgs lists of a scene dict (renderer.make_scene's band-count fields)."""
    ndc = bool(scene.get("use_ndc"))
    p, d = int(scene.get("n_freq_pos", 10)), int(scene.get("n_freq_dir", 4))
    p0, d0 = scene.get("n_freq_pos0"), scene.get("n_freq_dir0")
    p0 = (2 if ndc else p) if p0 is None or p0 == 0 else int(p0)
    d0 = (2 if ndc else d) if d0 is None or d0 == 0 else int(d0)
    def entry(a, b):
        if a < 0 and b < 0:
            return "none", "10-4"    # NoEncoding ignores posEncArgs
        return "nerf", f"{max(a, 0)}-{max(b, 0)}"
    (e0, a0), (e1, a1) = entry(p0, d0), entry(p, d)
    return f"[{e0}, {e1}]", f"[{a0}, {a1}]"


# losses[0] of a FromClassifiedDepth run -> the transform its sampler applies to raw0 (src/nerf_raymarch_common.py:625-637),
# as option "pdf_transform" numbers it
PDF_TRANSFORMS = {"BCEWithLogitsLoss": 1, "CrossEntropyLoss": 2, "CrossEntropyLossWeighted": 2}


def export_sampler(path):
    """(sampler, pdf_transform) of an export directory's config.ini, as adn_create_from_export_dir sets options "sampler" and
    "pdf_transform": (0, None) for the adaptive samplers, (1, 1 or 2) for FromClassifiedDepth, (2, None) for a one-network
    LinearlySpacedZNearZFar export.  Raises ValueError for a FromClassifiedDepth run whose losses[0] selects no transform."""
    import os
    cfg = {}
    with open(os.path.join(path, "config.ini")) as f:
        for line in f:
            if "=" in line and not line.lstrip().startswith(("#", ";")):
                k, v = line.split("=", 1)
                cfg[k.strip()] = [x.strip() for x in v.strip().strip("[]").split(",")]
    if len(cfg.get("rayMarchSampler", [])) == 1:
        return 2, None
    if cfg.get("rayMarchSampler", [""])[-1] != "FromClassifiedDepth":
        return 0, None
    loss0 = cfg.get("losses", [""])[0]
    if loss0 not in PDF_TRANSFORMS:
        raise ValueError(f"{path}: FromClassifiedDepth with losses[0] = {loss0 or '(missing)'} applies no transform (not supported)")
    return 1, PDF_TRANSFORMS[loss0]


def write_export_dir(path, scene, sd0, sd1, thr, K, sampler="FromClassifiedDepthAdaptive", sampling_loss="BCEWithLogitsLoss"):
    """Writes {config.ini, dataset_info.txt, model0.onnx, model1.onnx} in the reference's export format
    (src/export.py:28-93, src/train_data.py:180-195), config.ini with the networks' layers / layerWidth / skips and the
    scene's posEnc / posEncArgs.  sampler: rayMarchSampler of the shading net, FromClassifiedDepthAdaptive or
    FromClassifiedDepth (not with NDC); for FromClassifiedDepth, sampling_loss is losses[0], which picks the transform of
    the sampling net's output (PDF_TRANSFORMS)."""
    if sampler not in ("FromClassifiedDepthAdaptive", "FromClassifiedDepth"):
        raise ValueError(f"write_export_dir: sampler {sampler!r} is not FromClassifiedDepthAdaptive or FromClassifiedDepth")
    if sampler == "FromClassifiedDepth" and (scene.get("use_ndc") or sampling_loss not in PDF_TRANSFORMS):
        raise ValueError("write_export_dir: FromClassifiedDepth needs a non-NDC scene and losses[0] in " + ", ".join(PDF_TRANSFORMS))
    import os
    os.makedirs(path, exist_ok=True)
    (d0, w0, _), (d1, w1, skip) = net_shapes(sd0, sd1)
    cells = int(sd0[f"layers.{d0 - 1}.weight"].shape[0])   # multiDepthFeatures: the sampling net's output width
    as_np = lambda sd: {k: (v.detach().cpu().numpy() if hasattr(v, "detach") else np.asarray(v)) for k, v in sd.items()}
    write_onnx_initializers(os.path.join(path, "model0.onnx"), as_np(sd0))
    write_onnx_initializers(os.path.join(path, "model1.onnx"), as_np(sd1))
    ndc = bool(scene.get("use_ndc"))
    with open(os.path.join(path, "dataset_info.txt"), "w") as f:
        f.write(f"view_cell_center = {list(scene['view_cell_center'])}\n")
        f.write(f"view_cell_size = {list(scene['view_cell_size'])}\n")
        f.write(f"depth_range = {list(scene['depth_range'])}\n")
        f.write(f"fov = {scene['fov']}\nfocal = 0.0\ncamera_scale = 1.0\nmax_depth = {scene['max_depth']}\n")
        if ndc and scene.get("w") and scene.get("h"):   # not written by src/export.py; read by our loader when present
            f.write(f"w = {int(scene['w'])}\nh = {int(scene['h'])}\n")
    pos_enc, pos_enc_args = _enc_entries(scene)
    with open(os.path.join(path, "config.ini"), "w") as f:
        f.write(f"posEnc = {pos_enc}\nposEncArgs = {pos_enc_args}\n")
        if ndc:   # configs/fine_training_ndc.ini
            f.write("inFeatures = [SpherePosDir, RayMarchFromPoses]\n"
                    "outFeatures = [RawSigmoid, RGBARayMarch]\nrayMarchSampler = [none, FromClassifiedDepthAdaptiveNoDepthRange]\n"
                    "rayMarchNormalization = [InverseSqrtDistCentered, None]\nuseNDC = True\n"
                    f"numRaymarchSamples = [{K}, {K}]\ndepthTransform = linear\nzNear = [0.001, 0.001]\nzFar = [1.0, 1.0]\n"
                    f"adaptiveSamplingThreshold = {thr}\nmultiDepthFeatures = [{cells}, {cells}]\naccumulationMult = alpha\n")
        else:
            f.write("inFeatures = [SpherePosDir, RayMarchFromPoses]\n"
                    f"outFeatures = [RawSigmoid, RGBARayMarch]\nrayMarchSampler = [none, {sampler}]\n"
                    "rayMarchNormalization = [InverseSqrtDistCentered, InverseSqrtDistCentered]\n"
                    f"numRaymarchSamples = [{K}, {K}]\ndepthTransform = log\nzNear = [0.001, 0.001]\nzFar = [1.0, 1.0]\n"
                    f"adaptiveSamplingThreshold = {thr}\nmultiDepthFeatures = [{cells}, {cells}]\naccumulationMult = alpha\n")
            if sampler == "FromClassifiedDepth":
                f.write(f"losses = [{sampling_loss}, MSE]\n")
        f.write(f"activation = [relu, nerf]\nlayers = [{d0}, {d1}]\nlayerWidth = [{w0}, {w1}]\nskips = [, {_skips_entry(d1, skip)}]\n")


def write_nerf_export_dir(path, scene, sd, K):
    """Writes {config.ini, dataset_info.txt, model0.onnx} of a one-network run (plain NeRF: inFeatures =
    [RayMarchFromPoses], rayMarchSampler = [LinearlySpacedZNearZFar], or on NDC scenes [LinearlySpacedZNearZFarNoDepthRange]
    with rayMarchNormalization [None]), config.ini with one-item lists.  sd: the NeRF net (pts_linears.*).  The scene's
    depth_range goes to dataset_info.txt as it is: the renderer warps the depths with it (see INTEGRATION.md on which range
    a run uses)."""
    import os
    os.makedirs(path, exist_ok=True)
    d1, w1, skip = shading_shape(sd)
    write_onnx_initializers(os.path.join(path, "model0.onnx"),
                            {k: (v.detach().cpu().numpy() if hasattr(v, "detach") else np.asarray(v)) for k, v in sd.items()})
    ndc = bool(scene.get("use_ndc"))
    with open(os.path.join(path, "dataset_info.txt"), "w") as f:
        f.write(f"view_cell_center = {list(scene['view_cell_center'])}\n")
        f.write(f"view_cell_size = {list(scene['view_cell_size'])}\n")
        f.write(f"depth_range = {list(scene['depth_range'])}\n")
        f.write(f"fov = {scene['fov']}\nfocal = 0.0\ncamera_scale = 1.0\nmax_depth = {scene['max_depth']}\n")
        if ndc and scene.get("w") and scene.get("h"):
            f.write(f"w = {int(scene['w'])}\nh = {int(scene['h'])}\n")
    pos_enc, pos_enc_args = (e.strip("[]").split(", ")[-1] for e in _enc_entries(scene))
    zn, zf = float(scene.get("z_near", 0.001)), float(scene.get("z_far", 1.0))
    with open(os.path.join(path, "config.ini"), "w") as f:
        f.write(f"posEnc = [{pos_enc}]\nposEncArgs = [{pos_enc_args}]\ninFeatures = [RayMarchFromPoses]\noutFeatures = [RGBARayMarch]\n")
        if ndc:
            f.write("rayMarchSampler = [LinearlySpacedZNearZFarNoDepthRange]\nrayMarchNormalization = [None]\nuseNDC = True\n"
                    "depthTransform = linear\n")
        else:
            f.write("rayMarchSampler = [LinearlySpacedZNearZFar]\nrayMarchNormalization = [InverseSqrtDistCentered]\n"
                    "depthTransform = log\n")
        f.write(f"numRaymarchSamples = [{K}]\nzNear = [{zn}]\nzFar = [{zf}]\nactivation = [nerf]\nlosses = [MSE]\n"
                f"layers = [{d1}]\nlayerWidth = [{w1}]\nskips = [{_skips_entry(d1, skip)}]\n")
