"""CPU tests of oracle/mlp_emulation.py: the bf16-faithful emulation implements the same networks as the fp64 oracle,
the exactly-summing networks satisfy the conditions their bit-exact GPU comparison rests on, and that comparison has
teeth -- a one-step change of any weight tensor, a bias, a head weight, or a dropped lo*hi product changes the output."""
import numpy as np
import pytest
import torch

from conftest import case_weights, load_golden
from oracle import adanerf_oracle as orc
from oracle import mlp_emulation as me

ROWS = 512


def _x0(case):
    return torch.from_numpy(load_golden(case)["x0"][:ROWS])


def _x1(case):
    g = load_golden(case)
    mask = np.isfinite(g["z_nan"]).flatten()
    return torch.from_numpy(g["x1_nan"].reshape(-1, 90)[mask][:ROWS])


@pytest.mark.parametrize("case", ["pav_k8_t0.2", "shaped_k8_t0.2", "rand_k8_t0.2"])
@pytest.mark.parametrize("terms", [1, 3])
def test_mlp0_emulation_is_the_oracle_network(case, terms):
    """Same network as orc.mlp0_forward: bf16 operands (~2^-9 per operand) for terms = 1, fp32 class for terms = 3."""
    sd0, _ = case_weights(case)
    x0 = _x0(case)
    ref = orc.mlp0_forward(x0.double(), orc.to_dtype(sd0, torch.float64))
    emu = me.mlp0_emulate(x0, sd0, terms=terms)
    assert emu.dtype == torch.float32 and emu.shape == ref.shape
    rel = float((emu.double() - ref).abs().max() / ref.abs().max())
    assert rel < (2.0 ** -14 if terms == 3 else 2.0 ** -5), rel


@pytest.mark.parametrize("case", ["pav_k8_t0.2", "shaped_k8_t0.2", "rand_k8_t0.2"])
def test_mlp1_emulation_is_the_oracle_network(case):
    """Same network as orc.mlp1_forward (skip, feature / views wiring, heads): every output column within bf16 bounds."""
    _, sd1 = case_weights(case)
    x1 = _x1("shaped_k8_t0.2" if case.startswith("rand") else case)
    ref = orc.mlp1_forward(x1.double(), orc.to_dtype(sd1, torch.float64))
    emu = me.mlp1_emulate(x1, sd1)
    rel = (emu.double() - ref).abs().amax(0) / ref.abs().amax(0)
    assert bool((rel < 2.0 ** -5).all()), rel.tolist()
    # chunking changes nothing
    assert torch.equal(me.mlp1_emulate(x1, sd1, chunk_rows=100), emu)


def test_split_matches_the_packing():
    """hi = RNE bf16, lo = bf16(x - hi): the values pack_layer / pack_rows / the epilogue store."""
    x = torch.tensor([1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -9, 257.0, 4095.0, -3.14159265, 2.0 ** -20 * 5])
    hi, lo = me.split(x, 2)
    assert hi.tolist() == [1.0, 1.0 + 2.0 ** -7, 256.0, 4096.0, -3.140625, 2.0 ** -20 * 5]
    assert lo.tolist()[:4] == [2.0 ** -8, -(2.0 ** -9), 1.0, -1.0]
    assert (hi + lo - x.double()).abs().max() < 2.0 ** -16 * 4


@pytest.mark.parametrize("terms", [1, 3])
@pytest.mark.parametrize("shape", me.EXACT_SAMPLING_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_exact_sampling_nets_pass_their_self_check(shape, terms):
    n_in, depth, n_out = shape
    sd, x = me.exact_sampling_net(n_in, depth, n_out, terms, rows=1024)
    assert x.shape == (1024, n_in) and sd[f"layers.{depth - 1}.weight"].shape == (n_out, 256 if depth > 1 else n_in)
    again, x2 = me.exact_sampling_net(n_in, depth, n_out, terms, rows=700)     # deterministic; a prefix of the longer set
    assert all(torch.equal(sd[k], again[k]) for k in sd) and torch.equal(x[:700], x2)


def test_exact_shading_net_passes_its_self_check():
    sd, x = me.exact_shading_net(rows=1024)
    assert x.shape == (1024, 90) and sd["pts_linears.5.weight"].shape == (256, 319)
    assert sd["views_linears.0.weight"].shape == (128, 283)


def test_self_check_rejects_an_inexact_network():
    sd, x = me.exact_sampling_net(90, 2, 128, 3, rows=ROWS)
    bad = dict(sd)
    bad["layers.1.weight"] = sd["layers.1.weight"] * 2.0 ** 12     # sums far above 2^24 Q
    with pytest.raises(me.NotExact, match="2\\^24"):
        me.check_sampling_exact(bad, x, 3)
    dead = dict(sd)
    dead["layers.0.bias"] = sd["layers.0.bias"] - 1e6                # every unit zero on every row
    with pytest.raises(me.NotExact):
        me.check_sampling_exact(dead, x, 3)


# ------------------------------------------------------------------------------------------------------------- teeth
def _bf16_ulp(w):
    return 2.0 ** (np.floor(np.log2(abs(w))) - 7)


def _bumped(sd, key, reach, split=False):
    """sd with the weight of `key` that reaches the output most moved by the smallest step the kernel can see: one bf16
    ulp, or for the split net one ulp of hi + lo (bf16 ulp * 2^-8)."""
    W = sd[key].clone()
    r = reach.cpu() * (W != 0)
    row, col = np.unravel_index(int(r.flatten().argmax()), W.shape)
    w = float(W[row, col])
    W[row, col] = w + _bf16_ulp(w) * (2.0 ** -8 if split else 1.0)
    return dict(sd, **{key: W})


def _bias_bumped(sd, key, reach, scale):
    """sd with the bias of `key` that reaches the output most moved by one bf16 ulp of its unit's largest activation."""
    b = sd[key].clone()
    i = int(reach.cpu().argmax())
    b[i] += float(_bf16_ulp(max(1.0, float(scale[i]))))
    return dict(sd, **{key: b})


@pytest.mark.parametrize("terms", [1, 3])
@pytest.mark.parametrize("shape", [(90, 8, 128), (17, 2, 128)], ids=lambda s: "x".join(map(str, s)))
def test_teeth_sampling(shape, terms):
    n_in, depth, n_out = shape
    sd, x = me.exact_sampling_net(n_in, depth, n_out, terms)
    reach = me.check_sampling_exact(sd, x, terms)
    base, vals = me.mlp0_emulate(x, sd, terms=terms, trace=True)
    for l in range(depth):
        key = f"layers.{l}.weight"
        assert not torch.equal(me.mlp0_emulate(x, _bumped(sd, key, reach["weight"][l], terms == 3), terms=terms), base), key
        bumped = _bias_bumped(sd, f"layers.{l}.bias", reach["bias"][l], vals[l].abs().amax(0))
        assert not torch.equal(me.mlp0_emulate(x, bumped, terms=terms), base), f"layers.{l}.bias"
    if terms == 3:
        for drop in ("lh", "hl"):
            prods = tuple(p for p in me.TERMS3 if p != drop)
            assert not torch.equal(me.mlp0_emulate(x, sd, products=prods), base), drop


def test_teeth_shading():
    sd, x = me.exact_shading_net()
    reach = me.check_shading_exact(sd, x)
    base, vals = me.mlp1_emulate(x, sd, trace=True)
    names = [f"pts_linears.{i}" for i in range(8)] + ["feature_linear", "views_linears.0"]
    for i, name in enumerate(names):
        key = name + ".weight"
        assert not torch.equal(me.mlp1_emulate(x, _bumped(sd, key, reach[key])), base), key
        bumped = _bias_bumped(sd, name + ".bias", reach[name + ".bias"], vals[i].abs().amax(0))
        assert not torch.equal(me.mlp1_emulate(x, bumped), base), name + ".bias"
    for key in ("alpha_linear.weight", "rgb_linear.weight"):
        assert not torch.equal(me.mlp1_emulate(x, _bumped(sd, key, reach[key])), base), key
    # the view features 16..26 (what a floor instead of a ceiling K-step count would drop) reach the output
    x2 = x.clone()
    x2[:, 63 + 16:] = 0.0
    assert not torch.equal(me.mlp1_emulate(x2, sd), base)
