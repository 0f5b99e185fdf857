"""bf16-faithful emulation of the two MLP kernels (csrc/mlp.cu) and generators of exactly-summing test networks.

TEST INFRASTRUCTURE, NOT PRODUCT CODE.  `adanerf_oracle.mlp0_forward` / `mlp1_forward` state what the networks compute;
this module states how the kernel computes it, step by step:

  * every GEMM operand (the packed inputs, the weights of `pack_layer`, the inter-layer activations) is rounded to bf16
    with round-to-nearest-even, zero padded;
  * the split-precision sampling net (mlp0_terms = 3) splits each operand into hi = bf16(x), lo = bf16(x - hi) and sums
    hi*hi + lo*hi + hi*lo (lo*lo is not formed);
  * the products are accumulated (here in float64), rounded to fp32, the fp32 bias is added in fp32, then ReLU;
  * the shading net's heads are fp32 dot products of fp32 post-ReLU values (layer 7 -> alpha, the views layer -> rgb).

Plain torch on any device: the GPU tests run it in float64 on the device.  When every accumulation is exact in fp32
(the networks of `exact_sampling_net` / `exact_shading_net`), the kernel's output equals `mlp0_emulate` / `mlp1_emulate`
bit for bit, whatever order the tensor cores add in.
"""
import math

import torch

TERMS3 = ("hh", "lh", "hl")   # products of the split net: a_hi*w_hi, a_lo*w_hi, a_hi*w_lo
_PART = {"h": 0, "l": 1}


def bf16(x):
    """Round-to-nearest-even to bf16 of the fp32 value of x, returned in x's dtype."""
    return x.to(torch.float32).to(torch.bfloat16).to(x.dtype)


def split(x, nsplit):
    """(hi,) or (hi, lo) with hi = bf16(x), lo = bf16(fp32(x - hi)), as pack_layer / pack_rows / the epilogue form them."""
    x32 = x.to(torch.float32)
    hi = bf16(x32)
    if nsplit == 1:
        return (hi.double(),)
    return hi.double(), bf16(x32 - hi).double()


def _linear(a_parts, w_parts, b, products):
    """fp32(sum of the products, accumulated in float64) + fp32 bias, in fp32."""
    acc = None
    for p in products:
        t = a_parts[_PART[p[0]]] @ w_parts[_PART[p[1]]].T
        acc = t if acc is None else acc + t
    return acc.to(torch.float32) + b.to(device=acc.device, dtype=torch.float32)


def _chunks(n, chunk_rows):
    step = n if not chunk_rows else int(chunk_rows)
    for r0 in range(0, n, max(step, 1)):
        yield slice(r0, min(n, r0 + step))


def _products(terms, products):
    if products is not None:
        return tuple(products)
    if terms not in (1, 3):
        raise ValueError("terms must be 1 or 3")
    return TERMS3 if terms == 3 else ("hh",)


def mlp0_emulate(x0, sd0, terms=3, products=None, chunk_rows=None, trace=False):
    """Sampling net (BaseNet, ReLU between layers, raw last layer) as mlp_kernel<NSPLIT = 1 or 2> computes it.
    x0 [N, n_in] -> raw0 [N, n_out] fp32 on x0's device.  products: override the split net's product set (tests).
    trace: also return the per-layer fp32 values (pre-bf16, post-ReLU) of the first chunk."""
    prods = _products(terms, products)
    nsplit = 2 if any("l" in p for p in prods) else 1
    dev = x0.device
    D = len([k for k in sd0 if k.startswith("layers.") and k.endswith(".weight")])
    Ws = [split(sd0[f"layers.{l}.weight"].to(dev), nsplit) for l in range(D)]
    bs = [sd0[f"layers.{l}.bias"].to(device=dev, dtype=torch.float32) for l in range(D)]
    outs, tr = [], []
    for sl in _chunks(x0.shape[0], chunk_rows):
        a = split(x0[sl], nsplit)
        for l in range(D):
            v = _linear(a, Ws[l], bs[l], prods)
            if l + 1 < D:
                v = torch.clamp_min(v, 0.0)
                a = split(v, nsplit)
            if trace and not outs:
                tr.append(v)
        outs.append(v)
    out = torch.cat(outs, 0)
    return (out, tr) if trace else out


SHADING_LAYERS = [f"pts_linears.{i}" for i in range(8)] + ["feature_linear", "views_linears.0"]
SHADING_HEADS = (("alpha_linear", 7), ("rgb_linear", 9))   # head, layer whose fp32 post-ReLU values it reads


def _shading_walk(x, linear, rnd, upto=len(SHADING_LAYERS)):
    """The layer program build_net1 lays out, the one place it is written down here: pts = rnd(x[:, :63]) and
    views = rnd(x[:, 63:90]); layer 5 reads cat[pts, h], views_linears (layer 9) reads cat[feature, views]; every layer
    but feature_linear (layer 8) has a ReLU; the next layer reads rnd(value).  linear(i, inp) gives layer i's
    pre-activation.  Returns (input, pre-activation, value) per layer."""
    pts, views = rnd(x[:, :63]), rnd(x[:, 63:90])
    h, out = pts, []
    for i in range(upto):
        inp = torch.cat([pts, h], -1) if i == 5 else (torch.cat([h, views], -1) if i == 9 else h)
        pre = linear(i, inp)
        v = pre if i == 8 else torch.clamp_min(pre, 0.0)
        out.append((inp, pre, v))
        h = rnd(v)
    return out


def _shading_linear(sd1, dev):
    """linear(i, inp) of the kernel: bf16 weights, float64 accumulation rounded to fp32, + the fp32 bias in fp32."""
    W = {}

    def linear(i, inp):
        name = SHADING_LAYERS[i]
        if name not in W:
            W[name] = split(sd1[name + ".weight"].to(dev), 1)
        return _linear((inp,), W[name], sd1[name + ".bias"], ("hh",))
    return linear


def _bf16_f64(t):
    return bf16(t.to(torch.float32)).double()


def mlp1_emulate(x1, sd1, chunk_rows=None, trace=False):
    """Shading net (NeRF D=8 W=256 skip 4, use_viewdirs) as mlp_kernel<1> runs build_net1's program (`_shading_walk`),
    with alpha = fp32(<layer 7's fp32 post-ReLU row, alpha_w>) + alpha_b and rgb = fp32(<views layer's fp32 post-ReLU
    row, rgb_w>) + rgb_b.  x1 [M, 90] -> raw1 [M, 4] = [rgb, alpha] fp32.  trace: also the per-layer fp32 values of the
    first chunk (post-ReLU; feature_linear's without one)."""
    dev = x1.device
    linear = _shading_linear(sd1, dev)
    outs, tr = [], []
    for sl in _chunks(x1.shape[0], chunk_rows):
        vals = _shading_walk(x1[sl], linear, _bf16_f64)
        heads = {}
        for key, l in SHADING_HEADS:
            w = sd1[key + ".weight"].to(device=dev, dtype=torch.float32).double()
            heads[key] = (vals[l][2].double() @ w.T).to(torch.float32) + sd1[key + ".bias"].to(device=dev, dtype=torch.float32)
        outs.append(torch.cat([heads["rgb_linear"], heads["alpha_linear"]], -1))
        if trace and len(outs) == 1:
            tr = [v for _, _, v in vals]
    out = torch.cat(outs, 0)
    return (out, tr) if trace else out


# ----------------------------------------------------------------------------------------------------------------------
# exactly-summing networks
# ----------------------------------------------------------------------------------------------------------------------
EXACT_LIMIT = 2.0 ** 24
_BUDGET = 2.0 ** 22          # design-time bound on sum |terms| of one output element (the check allows 2^24 * Q)
_IN_MAX = 4095               # integer inputs below 2^12: at most 12 significant bits, so their hi / lo split is exact


# The exactly-summing networks the kernel tests run: sampling nets (n_in, depth, n_out) with mlp0_terms 1 and 3 -- one
# layer with 128 outputs (2 ring stages per tile, so alternate tiles of a CTA start on the other ring phase) and with 256,
# 8 and 12 layers, and two layers over every input width class (one K step, a partial second K step, two blocks ...).
EXACT_SAMPLING_SHAPES = [(90, 1, 128), (90, 1, 256), (90, 8, 128), (90, 12, 256)] + [
    (w, 2, 128) for w in (1, 16, 17, 30, 63, 64, 65, 90, 128)]


class NotExact(AssertionError):
    """A generated network / input set fails one of the conditions its bit-exact comparison rests on."""


def _quantum(*ts):
    """Largest power of two that divides every element of the tensors (inf when all are zero)."""
    q = math.inf
    for t in ts:
        t = t[t != 0].double()
        if t.numel() == 0:
            continue
        m, e = torch.frexp(t)
        mi = (m.abs() * 2.0 ** 53).to(torch.int64)
        low = (mi & -mi).double()
        k = e.to(torch.int64) - 53 + torch.log2(low).round().to(torch.int64)
        q = min(q, 2.0 ** int(k.min()))
    return q


def _rand_int(g, shape, lo, hi):
    return torch.randint(lo, hi + 1, shape, generator=g).to(torch.float32)


def _inputs(seed, rows, n_in, block=512):
    """Integer input rows below 2^12 in magnitude, drawn block by block so that fewer rows are a prefix of more."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(0, rows, block):
        x = _rand_int(g, (block, n_in), 1, _IN_MAX) * (torch.randint(0, 2, (block, n_in), generator=g) * 2 - 1).float()
        # sprinkle exact zeros and small values (exact in bf16) among the lo-carrying ones
        sel = torch.rand(block, n_in, generator=g)
        x = torch.where(sel < 0.03, torch.zeros_like(x), x)
        x = torch.where((sel >= 0.03) & (sel < 0.08), torch.round(x / 512), x)
        n_small = max(1, n_in // 8) if n_in > 1 else 0   # columns below 64 in magnitude: room for -257 weights
        if n_small:
            x[:, n_in - n_small:] = torch.round(x[:, n_in - n_small:] / 64)
        out.append(x)
    return torch.cat(out, 0)[:rows]


def _sparse_layer(g, n_out, n_in, U, allow_257, signed=False, busy=None, budget=_BUDGET):
    """Integer weights [n_out, n_in]: three nonzeros per row (fewer when n_in < 3), one positive and the rest negative.
    The positive weight is 2 on inputs below 2^12 and 1 above, which keeps the activations between a few hundred and a
    few ten thousand at any depth; the negative ones are -1 or -2, or -257 (a nonzero weight-lo part) when allow_257.
    Every input column is used by some row.  U [n_in]: the largest |input| seen per column, kept x2 below the budget.
    signed: the inputs take both signs (the network input), so -257 goes only on inputs below 2^7; on post-ReLU inputs
    it only lowers the unit, and any input within the budget (without the x2 margin: 2^22, a 4x margin to 2^24 that
    the check on the returned rows confirms) will do; of those the one nonzero on the fewest rows (busy [n_in]: that
    fraction), so the unit still passes its other inputs on most rows."""
    W = torch.zeros(n_out, n_in)
    k = min(3, n_in)
    cover = torch.randperm(n_in, generator=g)
    n_257 = 0
    for i in range(n_out):
        cols = [int(cover[s]) for s in range(i * k, min(n_in, i * k + k))]
        while len(cols) < k:
            c = int(torch.randint(0, n_in, (1,), generator=g))
            if c not in cols:
                cols.append(c)
        mags = []
        for t, c in enumerate(cols):
            m = 1.0 + float(torch.randint(0, 2, (1,), generator=g))
            if t == 0:
                m = 2.0 if float(U[c]) < 4096 else 1.0
            mags.append(m)
        # shrink magnitudes (257 first) until the row fits the budget
        for t in sorted(range(len(cols)), key=lambda t: -mags[t] * float(U[cols[t]])):
            if 2 * sum(m * float(U[c]) for m, c in zip(mags, cols)) <= budget:
                break
            mags[t] = 1.0
        if 2 * sum(m * float(U[c]) for m, c in zip(mags, cols)) > budget:
            raise NotExact(f"no exact weight row fits the budget (inputs up to {float(U.max()):.0f})")
        # one more input with weight -257 (hi -256, lo -1) on about one row in twelve, and on the last rows until the
        # layer has four: the least busy of a few candidates that fits
        if allow_257 and (float(torch.rand(1, generator=g)) < 0.08 or n_out - i <= 4 - n_257):
            cand = [c for c in torch.randint(0, n_in, (32,), generator=g).tolist() if c not in cols]
            base = sum(m * float(U[x]) for m, x in zip(mags, cols))
            fits = [c for c in cand if ((257.0 * float(U[c]) <= 2.0 ** 15) if signed else (base + 257.0 * float(U[c]) <= budget))]
            if fits:
                cols.append(min(fits, key=lambda x: (0.0 if busy is None else float(busy[x]), float(U[x]))))
                mags.append(257.0)
                n_257 += 1
        for t, (m, c) in enumerate(zip(mags, cols)):
            W[i, c] = m if t == 0 else -m
    return W


def _median_bias(pre, W):
    """Integer bias that puts the unit's zero crossing at the median pre-activation of the calibration rows: the unit is
    zero on about half of them, and its positive values span at most the spread of its pre-activation.  Units with a
    -257 weight get no positive bias: their median lies far below zero, and lifting it would scale them up 257x."""
    b = 1.0 - torch.round(pre.double().median(0).values).cpu()   # + 1: an odd offset, so sums of bf16 values need rounding
    big = (W.abs() > 2).any(1)
    return torch.where(big, torch.clamp_max(b, 0.0), b).to(torch.float32)


def _col_max(v):
    return v.double().abs().amax(0).cpu()


def exact_sampling_net(n_in=90, depth=8, n_out=128, terms=3, rows=2048, seed=0, device="cpu", calib_rows=2048):
    """Deterministic sampling net and input rows whose fp32 accumulation is exact in any order (see `check_sampling_exact`).
    Returns (sd0 with float32 CPU tensors, x0 [rows, n_in] float32 on `device`).  The biases are set on the first
    calib_rows rows, so a longer input set with the same seed extends a shorter one with the same network.  The checks
    run on the returned rows together with the calibration rows."""
    g = torch.Generator().manual_seed(1000003 * seed + 7919 * depth + 131 * n_in + n_out + terms)
    nsplit = 2 if terms == 3 else 1
    x = _inputs(1000003 * seed + n_in, max(rows, calib_rows), n_in)
    xc = x[:calib_rows].to(device)
    U, busy = _col_max(xc), None
    sd = {}
    for l in range(depth):
        last = l == depth - 1
        W = _sparse_layer(g, n_out if last else 256, n_in if l == 0 else 256, U, allow_257=(nsplit == 2), signed=(l == 0),
                          busy=busy)
        sd[f"layers.{l}.weight"] = W
        sd[f"layers.{l}.bias"] = torch.zeros(W.shape[0])
        b = _rand_int(g, (W.shape[0],), -64, 64) if last else _median_bias(_pre_activation(xc, sd, l, terms), W)
        sd[f"layers.{l}.bias"] = b
        if not last:
            v = torch.clamp_min(_pre_activation(xc, sd, l, terms), 0.0)
            U, busy = _col_max(v), (v != 0).double().mean(0).cpu()
    x = x.to(device)
    check_sampling_exact(sd, x, terms)
    return sd, x[:rows]


def _pre_activation(x0, sd0, l, terms):
    """Layer l's fp32 pre-activation (accumulation + bias, before ReLU) on x0 with the layers 0..l of sd0."""
    sub = {k: v for k, v in sd0.items() if int(k.split(".")[1]) <= l}
    # emulate the prefix as a network whose last layer is l (the last layer of mlp0_emulate has no ReLU)
    return mlp0_emulate(x0, sub, terms=terms)


def exact_shading_net(rows=2048, seed=0, device="cpu", calib_rows=2048):
    """Deterministic shading net (full build_net1 shapes) and input rows x1 [rows, 90] whose fp32 accumulations, heads
    included, are exact in any order (see `check_shading_exact`).  Returns (sd1 float32 CPU tensors, x1 on `device`)."""
    g = torch.Generator().manual_seed(2000003 * seed + 17)
    x = _inputs(2000003 * seed + 90, max(rows, calib_rows), 90)
    xc = x[:calib_rows].to(device)
    P = torch.full((63,), float(_IN_MAX), dtype=torch.float64)
    V = torch.full((27,), float(_IN_MAX), dtype=torch.float64)
    sd = {}
    U = P
    for li, name in enumerate(SHADING_LAYERS):
        n_out = 128 if li == 9 else 256
        Uin = torch.cat([P, U]) if li == 5 else (torch.cat([U, V]) if li == 9 else U)
        W = _sparse_layer(g, n_out, Uin.numel(), Uin, allow_257=False)
        sd[name + ".weight"] = W
        sd[name + ".bias"] = torch.zeros(n_out)
        pre = _shading_walk(xc, _shading_linear(sd, xc.device), _bf16_f64, upto=li + 1)[li][1]
        b = _median_bias(pre, W) if li != 8 else _rand_int(g, (n_out,), -64, 64)
        sd[name + ".bias"] = b
        U = _col_max(_shading_walk(xc, _shading_linear(sd, xc.device), _bf16_f64, upto=li + 1)[li][2])
    sd["alpha_linear.weight"] = _signed_small(g, (1, 256))
    sd["alpha_linear.bias"] = _rand_int(g, (1,), -64, 64)
    sd["rgb_linear.weight"] = _signed_small(g, (3, 128))
    sd["rgb_linear.bias"] = _rand_int(g, (3,), -64, 64)
    x = x.to(device)
    check_shading_exact(sd, x)
    return sd, x[:rows]


def _signed_small(g, shape):
    return _rand_int(g, shape, 1, 2) * (torch.randint(0, 2, shape, generator=g) * 2 - 1).float()


# ----------------------------------------------------------------------------------------------------------------------
# self-checks
# ----------------------------------------------------------------------------------------------------------------------
def _check_layer(name, a_parts, w_parts, b, products):
    """Exactness bound of one layer: sum |terms| + |b| < 2^24 Q for every output element, Q the common quantum."""
    q = _quantum(b)
    s = b.double().abs().to(a_parts[0].device)
    for p in products:
        a, w = a_parts[_PART[p[0]]], w_parts[_PART[p[1]]]
        if a.abs().max() == 0 or w.abs().max() == 0:
            continue
        q = min(q, _quantum(a) * _quantum(w))
        s = s + a.abs() @ w.abs().T
    worst = float(s.max())
    if not worst < EXACT_LIMIT * q:
        raise NotExact(f"{name}: sum |terms| reaches {worst:.6g} >= 2^24 * Q (Q = {q:g})")
    return worst / q


def _check_relu_both_ways(name, v):
    pos = (v > 0).any(0)
    zero = (v <= 0).any(0)
    bad = ~(pos & zero)
    if bad.any():
        raise NotExact(f"{name}: {int(bad.sum())} units are never zero or never positive on these rows")


def _check_rounds(name, v, nsplit):
    big = v.abs() > 256
    inexact = bf16(v) != v
    if not (big & inexact).any():
        raise NotExact(f"{name}: no activation above 256 that bf16 rounds ({'no activation-lo part' if nsplit == 2 else 'rounding never acts'})")


def _check_effect(name, what, mask):
    if not bool(mask.all()):
        idx = torch.nonzero(~mask).flatten()[:8].tolist()
        raise NotExact(f"{name}: {what} {idx} ... have no effect on the output")


def _ste(fn):
    """Rounding with a straight-through gradient: the value of fn(x), the derivative of the identity."""
    return lambda x: x + (fn(x) - x).detach()


def check_sampling_exact(sd0, x0, terms):
    """Returns the reach of every weight and bias (|d output functional / d parameter| through these rows' ReLU masks).
    Raises NotExact unless, on the rows x0: every layer's accumulation is exact in any order (sum |terms| < 2^24 Q);
    every hidden unit is zero on some rows and positive on others; every input column, weight row and bias of every
    layer reaches the output; every hidden layer has activations above 256 that bf16 rounds; and for the split net the
    input and activation lo parts are nonzero, and so are the weight lo parts of every layer (but the first layer of a
    one-input net)."""
    nsplit = 2 if terms == 3 else 1
    prods = TERMS3 if nsplit == 2 else ("hh",)
    D = len([k for k in sd0 if k.endswith(".weight")])
    dev = x0.device
    a = split(x0, nsplit)
    if nsplit == 2 and not (a[1] != 0).any():
        raise NotExact("input lo parts are all zero")
    for l in range(D):
        W = split(sd0[f"layers.{l}.weight"].to(dev), nsplit)
        b = sd0[f"layers.{l}.bias"].to(dev)
        # every layer's hi*lo products see a nonzero weight lo -- but the first layer of a one-input net: its single
        # signed input column cannot also hold the small values a -257 weight needs
        if nsplit == 2 and not (W[1] != 0).any() and not (l == 0 and x0.shape[1] == 1):
            raise NotExact(f"layer {l}: the weight lo parts are all zero")
        _check_layer(f"layer {l}", a, W, b, prods)
        v = _linear(a, W, b, prods)
        if l + 1 < D:
            v = torch.clamp_min(v, 0.0)
            _check_relu_both_ways(f"layer {l}", v)
            _check_rounds(f"layer {l}", v, nsplit)
            a = split(v, nsplit)
    # reach: gradients of a generic linear functional of the output through the ReLU masks of these rows
    g = torch.Generator().manual_seed(1)
    xs = x0.double().clone().requires_grad_(True)
    r = _ste(lambda t: sum(split(t, nsplit)))
    h = r(xs)
    leaves, hs = [], [h]
    wleaves = []
    for l in range(D):
        W = sd0[f"layers.{l}.weight"].to(dev).double()
        W = sum(split(W, nsplit)).requires_grad_(True)
        wleaves.append(W)
        b = sd0[f"layers.{l}.bias"].to(dev).double().requires_grad_(True)
        leaves.append(b)
        pre = h @ W.T + b
        h = r(torch.clamp_min(pre, 0.0)) if l + 1 < D else pre
        if l + 1 < D:
            h.retain_grad()
            hs.append(h)
    c = torch.rand(h.shape[1], generator=g, dtype=torch.float64).to(dev) + 0.5
    (h * c).sum().backward()
    for l in range(D):
        _check_effect(f"layer {l}", "biases", leaves[l].grad != 0)
        inp = xs if l == 0 else hs[l]
        gin = xs.grad if l == 0 else hs[l].grad
        _check_effect(f"layer {l}", "input columns", ((inp * gin) != 0).any(0))
    # how strongly each weight / bias reaches the output (a first-order measure; tests pick what to perturb by it)
    return dict(weight=[w.grad.abs() for w in wleaves], bias=[b.grad.abs() for b in leaves])


def check_shading_exact(sd1, x1):
    """Returns the reach of every weight and bias by name (see `check_sampling_exact`), after checking
    the conditions of `check_sampling_exact` for the shading net (plain bf16), plus the heads: alpha and rgb are fp32
    dot products whose sums stay below 2^24 Q, and every head weight sees a nonzero input on some row."""
    dev = x1.device
    vals = _shading_walk(x1, _shading_linear(sd1, dev), _bf16_f64)
    for i, (name, (inp, _, v)) in enumerate(zip(SHADING_LAYERS, vals)):
        _check_layer(name, (inp,), split(sd1[name + ".weight"].to(dev), 1), sd1[name + ".bias"].to(dev), ("hh",))
        if i != 8:
            _check_relu_both_ways(name, v)
        if i != 9:
            _check_rounds(name, v, 1)
    for key, l in SHADING_HEADS:
        hv = vals[l][2]
        _check_layer(key, (hv.double(),), (sd1[key + ".weight"].to(dev).double(),), sd1[key + ".bias"].to(dev), ("hh",))
        _check_effect(key, "weights (columns never nonzero)", (hv != 0).any(0))
    # reach: the same program in float64 with straight-through rounding and parameter leaves
    leaves = {k: (bf16(v.to(dev).double()) if k.endswith(".weight") and not k.startswith(("alpha", "rgb")) else
                  v.to(dev).double()).requires_grad_(True) for k, v in sd1.items()}
    xs = x1.to(torch.float32).double().requires_grad_(True)
    vals = _shading_walk(xs, lambda i, inp: inp @ leaves[SHADING_LAYERS[i] + ".weight"].T + leaves[SHADING_LAYERS[i] + ".bias"],
                         _ste(bf16))
    for inp, _, _ in vals:
        inp.retain_grad()
    heads = {key: vals[l][2] @ leaves[key + ".weight"].T for key, l in SHADING_HEADS}
    c = torch.rand(4, generator=torch.Generator().manual_seed(2), dtype=torch.float64).to(dev) + 0.5
    (torch.cat([heads["rgb_linear"], heads["alpha_linear"]], -1) * c).sum().backward()
    for name, (inp, _, _) in zip(SHADING_LAYERS, vals):
        _check_effect(name, "biases", leaves[name + ".bias"].grad != 0)
        _check_effect(name, "input columns", ((inp * inp.grad) != 0).any(0))
    return {k: v.grad.abs() for k, v in leaves.items() if v.grad is not None}
