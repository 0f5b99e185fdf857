"""bf16-faithful emulation of the MLP kernels for networks of other shapes, and exactly-summing networks of those shapes.

TEST INFRASTRUCTURE, NOT PRODUCT CODE.  oracle/mlp_emulation.py emulates the kernels on the default shading net (8 x 256,
skip 4) and generates sampling nets with 256-wide hidden layers; this module states the layer program build_net1 lays out
for any supported shading net (D = 1-10 pts layers, W = 128 or 256, no skip or one) and generates exact networks of
those shapes and sampling nets with 128-wide hidden layers.  The arithmetic (bf16 rounding, float64 accumulation rounded
to fp32, fp32 bias and heads) and the self-checks are mlp_emulation's, reused as they are.  mlp_emulation.mlp0_emulate and
check_sampling_exact already handle any sampling-net width.
"""
import torch

from . import mlp_emulation as me
from .shape_oracle import shading_shape

DEFAULT_SHADING_SHAPE = (8, 256, 4)   # (D, W, skip) of NeRF(D=8, W=256, skips=[4])

# Sampling nets with 128-wide hidden layers, (n_in, depth, n_out, width): one N half per hidden layer, two activation
# blocks written in place; the NDC configs' 30 inputs; the deepest net.
EXACT_SAMPLING_SHAPES_W128 = [(90, 2, 128, 128), (90, 6, 128, 128), (30, 8, 128, 128), (128, 3, 256, 128), (90, 12, 128, 128)]
# Shading nets other than 8 x 256 / skip 4, (D, W, skip): the 6 x 128 skip-3 and 10 x 256 skip-4 nets, no skip (V loaded
# after layer 0), a skip after layer 0, a skip into the last pts layer (which also forms alpha), a one-layer net.
EXACT_SHADING_SHAPES = [(6, 128, 3), (8, 128, 4), (4, 256, -1), (10, 256, 4), (2, 128, 0), (5, 256, 3), (1, 128, -1)]


def shading_layers(D):
    """Names of the D + 2 GEMM layers of a shading net with D pts layers, in program order."""
    return [f"pts_linears.{i}" for i in range(D)] + ["feature_linear", "views_linears.0"]


def shading_heads(D):
    """(head, layer whose fp32 post-ReLU values it reads): alpha after the last pts layer, rgb after the view layer."""
    return (("alpha_linear", D - 1), ("rgb_linear", D + 1))


def shading_walk(x, linear, rnd, shape, upto=None):
    """The layer program build_net1 lays out for shape = (D, W, skip): pts = rnd(x[:, :63]) and views = rnd(x[:, 63:90]);
    the skip consumer (layer skip + 1, none when skip < 0) reads cat[pts, h], views_linears (layer D + 1) reads
    cat[feature, views]; every layer but feature_linear (layer D) has a ReLU; the next layer reads rnd(value).
    linear(i, inp) gives layer i's pre-activation.  Returns (input, pre-activation, value) of the first `upto` layers
    (default all)."""
    D, _, skip = shape
    pts, views = rnd(x[:, :63]), rnd(x[:, 63:90])
    h, out = pts, []
    for i in range(D + 2 if upto is None else upto):
        inp = torch.cat([pts, h], -1) if (skip >= 0 and i == skip + 1) else (torch.cat([h, views], -1) if i == D + 1 else h)
        pre = linear(i, inp)
        v = pre if i == D else torch.clamp_min(pre, 0.0)
        out.append((inp, pre, v))
        h = rnd(v)
    return out


def _shading_linear(sd1, dev, names):
    """linear(i, inp) of the kernel: bf16 weights, float64 accumulation rounded to fp32, + the fp32 bias in fp32."""
    W = {}

    def linear(i, inp):
        name = names[i]
        if name not in W:
            W[name] = me.split(sd1[name + ".weight"].to(dev), 1)
        return me._linear((inp,), W[name], sd1[name + ".bias"], ("hh",))
    return linear


def mlp1_emulate(x1, sd1, chunk_rows=None):
    """Shading net of any supported shape as mlp_kernel<1> runs build_net1's program (`shading_walk`), with
    alpha = fp32(<the last pts layer's fp32 post-ReLU row, alpha_w>) + alpha_b and rgb = fp32(<views layer's fp32
    post-ReLU row, rgb_w>) + rgb_b.  x1 [M, 90] -> raw1 [M, 4] = [rgb, alpha] fp32."""
    dev = x1.device
    shape = shading_shape(sd1)
    linear = _shading_linear(sd1, dev, shading_layers(shape[0]))
    outs = []
    for sl in me._chunks(x1.shape[0], chunk_rows):
        vals = shading_walk(x1[sl], linear, me._bf16_f64, shape)
        heads = {}
        for key, l in shading_heads(shape[0]):
            w = sd1[key + ".weight"].to(device=dev, dtype=torch.float32).double()
            heads[key] = (vals[l][2].double() @ w.T).to(torch.float32) + sd1[key + ".bias"].to(device=dev, dtype=torch.float32)
        outs.append(torch.cat([heads["rgb_linear"], heads["alpha_linear"]], -1))
    return torch.cat(outs, 0)


def exact_sampling_net(n_in=90, depth=6, n_out=128, terms=3, rows=2048, seed=0, device="cpu", calib_rows=2048, width=128):
    """mlp_emulation.exact_sampling_net with hidden layers `width` wide: a deterministic sampling net and input rows whose
    fp32 accumulation is exact in any order (mlp_emulation.check_sampling_exact)."""
    g = torch.Generator().manual_seed(1000003 * seed + 7919 * depth + 131 * n_in + n_out + terms + 17 * width)
    nsplit = 2 if terms == 3 else 1
    x = me._inputs(1000003 * seed + n_in, max(rows, calib_rows), n_in)
    xc = x[:calib_rows].to(device)
    U, busy = me._col_max(xc), None
    sd = {}
    for l in range(depth):
        last = l == depth - 1
        W = me._sparse_layer(g, n_out if last else width, n_in if l == 0 else width, U, allow_257=(nsplit == 2),
                             signed=(l == 0), busy=busy)
        sd[f"layers.{l}.weight"] = W
        sd[f"layers.{l}.bias"] = torch.zeros(W.shape[0])
        b = me._rand_int(g, (W.shape[0],), -64, 64) if last else me._median_bias(me._pre_activation(xc, sd, l, terms), W)
        sd[f"layers.{l}.bias"] = b
        if not last:
            v = torch.clamp_min(me._pre_activation(xc, sd, l, terms), 0.0)
            U, busy = me._col_max(v), (v != 0).double().mean(0).cpu()
    x = x.to(device)
    me.check_sampling_exact(sd, x, terms)
    return sd, x[:rows]


def exact_shading_net(shape, rows=2048, seed=0, device="cpu", calib_rows=2048):
    """Deterministic shading net of shape = (D, W, skip) and input rows x1 [rows, 90] whose fp32 accumulations, heads
    included, are exact in any order (see `check_shading_exact`), built like mlp_emulation.exact_shading_net.  Returns
    (sd1 float32 CPU tensors, x1 on `device`)."""
    D, Wd, skip = shape
    g = torch.Generator().manual_seed(2000003 * seed + 17 + 7919 * D + 131 * Wd + skip + 1)
    x = me._inputs(2000003 * seed + 90, max(rows, calib_rows), 90)
    xc = x[:calib_rows].to(device)
    P = torch.full((63,), float(me._IN_MAX), dtype=torch.float64)
    V = torch.full((27,), float(me._IN_MAX), dtype=torch.float64)
    names = shading_layers(D)
    sd = {}
    U = P
    for li, name in enumerate(names):
        n_out = Wd // 2 if li == D + 1 else Wd
        Uin = torch.cat([P, U]) if (skip >= 0 and li == skip + 1) else (torch.cat([U, V]) if li == D + 1 else U)
        W = me._sparse_layer(g, n_out, Uin.numel(), Uin, allow_257=False)
        sd[name + ".weight"] = W
        sd[name + ".bias"] = torch.zeros(n_out)
        pre = shading_walk(xc, _shading_linear(sd, xc.device, names), me._bf16_f64, shape, upto=li + 1)[li][1]
        sd[name + ".bias"] = me._median_bias(pre, W) if li != D else me._rand_int(g, (n_out,), -64, 64)
        U = me._col_max(shading_walk(xc, _shading_linear(sd, xc.device, names), me._bf16_f64, shape, upto=li + 1)[li][2])
    sd["alpha_linear.weight"] = me._signed_small(g, (1, Wd))
    sd["alpha_linear.bias"] = me._rand_int(g, (1,), -64, 64)
    sd["rgb_linear.weight"] = me._signed_small(g, (3, Wd // 2))
    sd["rgb_linear.bias"] = me._rand_int(g, (3,), -64, 64)
    x = x.to(device)
    check_shading_exact(sd, x)
    return sd, x[:rows]


def check_shading_exact(sd1, x1):
    """mlp_emulation.check_shading_exact for a shading net of any supported shape: on the rows x1, every layer's and
    head's accumulation is exact in any order; every hidden unit is zero on some rows and positive on others (but
    feature_linear's, which has no ReLU); every layer but the view layer has activations that bf16 rounds; every head
    weight sees a nonzero input; every input column and bias of every layer reaches the output.  Returns the reach of
    every parameter by name; raises mlp_emulation.NotExact."""
    dev = x1.device
    shape = shading_shape(sd1)
    D = shape[0]
    names, heads_of = shading_layers(D), shading_heads(D)
    vals = shading_walk(x1, _shading_linear(sd1, dev, names), me._bf16_f64, shape)
    for i, (name, (inp, _, v)) in enumerate(zip(names, vals)):
        me._check_layer(name, (inp,), me.split(sd1[name + ".weight"].to(dev), 1), sd1[name + ".bias"].to(dev), ("hh",))
        if i != D:
            me._check_relu_both_ways(name, v)
        if i != D + 1:
            me._check_rounds(name, v, 1)
    for key, l in heads_of:
        hv = vals[l][2]
        me._check_layer(key, (hv.double(),), (sd1[key + ".weight"].to(dev).double(),), sd1[key + ".bias"].to(dev), ("hh",))
        me._check_effect(key, "weights (columns never nonzero)", (hv != 0).any(0))
    # reach: the same program in float64 with straight-through rounding and parameter leaves
    leaves = {k: (me.bf16(v.to(dev).double()) if k.endswith(".weight") and not k.startswith(("alpha", "rgb")) else
                  v.to(dev).double()).requires_grad_(True) for k, v in sd1.items()}
    xs = x1.to(torch.float32).double().requires_grad_(True)
    vals = shading_walk(xs, lambda i, inp: inp @ leaves[names[i] + ".weight"].T + leaves[names[i] + ".bias"],
                        me._ste(me.bf16), shape)
    for inp, _, _ in vals:
        inp.retain_grad()
    heads = {key: vals[l][2] @ leaves[key + ".weight"].T for key, l in heads_of}
    c = torch.rand(4, generator=torch.Generator().manual_seed(2), dtype=torch.float64).to(dev) + 0.5
    (torch.cat([heads["rgb_linear"], heads["alpha_linear"]], -1) * c).sum().backward()
    for name, (inp, _, _) in zip(names, vals):
        me._check_effect(name, "biases", leaves[name + ".bias"].grad != 0)
        me._check_effect(name, "input columns", ((inp * inp.grad) != 0).any(0))
    return {k: v.grad.abs() for k, v in leaves.items() if v.grad is not None}
