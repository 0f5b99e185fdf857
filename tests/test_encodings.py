"""Positional encodings other than posEncArgs 10-4 (and 2-2 for the sampling net), without a GPU: the emulation of the
shading kernel for any position / view block width, the recurrence bound up to 20 bands, the export round trip of posEnc /
posEncArgs, check_state_dicts with an encoding and the adapter's reading of a TrainConfig's encodings.  The helpers here
are what tests/test_encodings_gpu.py compares the kernels against."""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import adanerf_oracle as orc
from oracle import mlp_emulation as me
from oracle import shape_oracle as so
from oracle import stage_emulation as se

# (name, scene fields, shading net shape (D, W, skip)) of the encodings tested end to end: both shading blocks at their
# limit with a two-block P through the skip consumer; the sampling format at its limit (126 columns); no encoding on either
# net; NDC with a two-block P.
CASES = [
    ("s10-4_p20-10", dict(n_freq_pos=20, n_freq_dir=10, n_freq_pos0=10, n_freq_dir0=4), (8, 256, 4)),
    ("s16-4_p6-2", dict(n_freq_pos=6, n_freq_dir=2, n_freq_pos0=16, n_freq_dir0=4), (8, 256, 4)),
    ("none", dict(n_freq_pos=-1, n_freq_dir=-1, n_freq_pos0=-1, n_freq_dir0=-1), (6, 128, 3)),
    ("ndc_s2-2_p12-6", dict(n_freq_pos=12, n_freq_dir=6, use_ndc=True, w=800, h=800), (8, 256, 4)),
]


def bands(scene):
    """((P0, D0), (P, D)) band counts of a scene dict as adn_create reads them (none / negative = 0 bands)."""
    p, d = scene.get("n_freq_pos", 10), scene.get("n_freq_dir", 4)
    ndc = bool(scene.get("use_ndc"))
    p0 = scene.get("n_freq_pos0") or (2 if ndc else p)
    d0 = scene.get("n_freq_dir0") or (2 if ndc else d)
    return (max(p0, 0), max(d0, 0)), (max(p, 0), max(d, 0))


def columns(scene):
    """(sampling-net inputs, shading-net position columns, view columns) of a scene dict."""
    (p0, d0), (p, d) = bands(scene)
    return 6 + 6 * (p0 + d0), 3 + 6 * p, 3 + 6 * d


def case_scene(fields):
    base = orc.SCENE_BARBERSHOP if fields.get("use_ndc") else orc.SCENE_PAVILLON
    return dict(base, **fields)


# ------------------------------------------------------------------------------------------- shading-net emulation
def shading_walk(x, linear, rnd, shape, n_p, n_v, upto=None):
    """shape_emulation.shading_walk with n_p position and n_v view columns: build_net1's layer program for any encoding."""
    D, _, skip = shape
    pts, views = rnd(x[:, :n_p]), rnd(x[:, n_p:n_p + n_v])
    h, out = pts, []
    for i in range(D + 2 if upto is None else upto):
        inp = torch.cat([pts, h], -1) if (skip >= 0 and i == skip + 1) else (torch.cat([h, views], -1) if i == D + 1 else h)
        pre = linear(i, inp)
        v = pre if i == D else torch.clamp_min(pre, 0.0)
        out.append((inp, pre, v))
        h = rnd(v)
    return out


def _linear_of(sd1, dev, names):
    W = {}

    def linear(i, inp):
        if names[i] not in W:
            W[names[i]] = me.split(sd1[names[i] + ".weight"].to(dev), 1)
        return me._linear((inp,), W[names[i]], sd1[names[i] + ".bias"], ("hh",))
    return linear


def mlp1_emulate(x1, sd1, n_p):
    """shape_emulation.mlp1_emulate for a shading net reading n_p position columns: x1 [M, n_p + n_v] -> raw1 [M, 4]."""
    shape = so.shading_shape(sd1, n_p)
    n_v = int(sd1["views_linears.0.weight"].shape[1]) - shape[1]
    names = [f"pts_linears.{i}" for i in range(shape[0])] + ["feature_linear", "views_linears.0"]
    vals = shading_walk(x1, _linear_of(sd1, x1.device, names), me._bf16_f64, shape, n_p, n_v)
    heads = {}
    for key, l in (("alpha_linear", shape[0] - 1), ("rgb_linear", shape[0] + 1)):
        w = sd1[key + ".weight"].to(device=x1.device, dtype=torch.float32).double()
        heads[key] = (vals[l][2].double() @ w.T).to(torch.float32) + sd1[key + ".bias"].to(device=x1.device, dtype=torch.float32)
    return torch.cat([heads["rgb_linear"], heads["alpha_linear"]], -1)


def exact_shading_net(shape, n_p, n_v, rows=2048, seed=0, device="cpu", calib_rows=2048):
    """shape_emulation.exact_shading_net with n_p position and n_v view columns: a shading net and input rows whose fp32
    accumulations are exact in any order, so the kernel must match mlp1_emulate bit for bit.  Checks that and returns
    (sd1, x1 [rows, n_p + n_v] on `device`)."""
    D, Wd, skip = shape
    g = torch.Generator().manual_seed(2000003 * seed + 17 + 7919 * D + 131 * Wd + skip + 1 + 31 * n_p + n_v)
    x = me._inputs(2000003 * seed + n_p + n_v, max(rows, calib_rows), n_p + n_v)
    xc = x[:calib_rows].to(device)
    P = torch.full((n_p,), float(me._IN_MAX), dtype=torch.float64)
    V = torch.full((n_v,), float(me._IN_MAX), dtype=torch.float64)
    names = [f"pts_linears.{i}" for i in range(D)] + ["feature_linear", "views_linears.0"]
    walk = lambda sd, upto: shading_walk(xc, _linear_of(sd, xc.device, names), me._bf16_f64, shape, n_p, n_v, upto=upto)
    sd, U = {}, P
    for li, name in enumerate(names):
        n_out = Wd // 2 if li == D + 1 else Wd
        Uin = torch.cat([P, U]) if (skip >= 0 and li == skip + 1) else (torch.cat([U, V]) if li == D + 1 else U)
        W = me._sparse_layer(g, n_out, Uin.numel(), Uin, allow_257=False)
        sd[name + ".weight"], sd[name + ".bias"] = W, torch.zeros(n_out)
        pre = walk(sd, li + 1)[li][1]
        sd[name + ".bias"] = me._median_bias(pre, W) if li != D else me._rand_int(g, (n_out,), -64, 64)
        U = me._col_max(walk(sd, li + 1)[li][2])
    sd["alpha_linear.weight"] = me._signed_small(g, (1, Wd))
    sd["alpha_linear.bias"] = me._rand_int(g, (1,), -64, 64)
    sd["rgb_linear.weight"] = me._signed_small(g, (3, Wd // 2))
    sd["rgb_linear.bias"] = me._rand_int(g, (3,), -64, 64)
    x = x.to(device)
    vals = shading_walk(x, _linear_of(sd, x.device, names), me._bf16_f64, shape, n_p, n_v)
    for i, (name, (inp, _, v)) in enumerate(zip(names, vals)):
        me._check_layer(name, (inp,), me.split(sd[name + ".weight"].to(x.device), 1), sd[name + ".bias"].to(x.device), ("hh",))
        if i != D:
            me._check_relu_both_ways(name, v)
    for key, l in (("alpha_linear", D - 1), ("rgb_linear", D + 1)):
        me._check_layer(key, (vals[l][2].double(),), (sd[key + ".weight"].to(x.device).double(),), sd[key + ".bias"].to(x.device), ("hh",))
    return sd, x[:rows]


# ---------------------------------------------------------------------------------------------- oracle composition
def oracle_render(pose, rot, dirs, sd0, sd1, scene, thr, K, return_stages=False):
    """adanerf_oracle.render_rays with the scene's encodings and a shading net of any shape (TrainConfig.inference,
    src/train_data.py:278-299).  posEnc none is posenc with 0 bands: the 3 inputs alone."""
    (p0, d0), (p, d) = bands(scene)
    ndc = bool(scene.get("use_ndc"))
    with torch.no_grad():
        x0, ray_o, ray_d = orc.stage0_sphere_pos_dir(pose, rot, dirs, scene, n_freq_pos=p0, n_freq_dir=d0)
        raw0 = orc.mlp0_forward(x0, sd0)
        s2 = orc.stage2_sample(raw0, thr, K, scene["depth_range"], no_depth_range=ndc)
        n = dirs.shape[0]
        dense = thr == 0.0
        x1, mapping, zs = orc.stage3_encode(ray_o, ray_d, s2["z"], scene, compact=not dense, n_freq_pos=p, n_freq_dir=d)
        raw1 = so.mlp1_forward(x1, sd1, input_ch=3 + 6 * p)
        comp = orc.stage5_composite(raw1, zs, s2["zp"], None if dense else mapping, n, K)
    out = dict(rgb=comp["rgb"], n_samples=mapping.view(n, K).sum(1))
    if return_stages:
        out.update(x0=x0, ray_o=ray_o, ray_d=ray_d, raw0=raw0, x1=x1, raw1=raw1)
    return out


def case_weights(scene, shape, seed=0, thr=0.2, K=8):
    """Reference-initialised nets for the scene's encodings (BaseNet / NeRF init order), the sampling net's last layer
    damped and shifted as make_weights("shaped") does, so that rays keep a ragged 1..K samples."""
    n0, n_p, n_v = columns(scene)
    D, Wd, skip = shape
    torch.manual_seed(seed)
    sd0 = orc.init_sampling_net(n_in=n0)
    sd1 = orc.init_shading_net(input_ch=n_p, input_ch_views=n_v, W=Wd, D=D, skips=(skip,) if skip >= 0 else ())
    sd0["layers.7.weight"] = sd0["layers.7.weight"] * 0.15
    sd0["layers.7.bias"] = sd0["layers.7.bias"] * 0.15 - 0.1
    for k in ("rgb_linear.weight", "alpha_linear.weight"):
        sd1[k] = sd1[k] * 0.05
    return sd0, sd1


# --------------------------------------------------------------------------------------------------------- tests
def test_recurrence_bound_holds_to_20_bands():
    """Every band stays within 1.7e-5 of float64 sin / cos, up to band 19, with anchors anywhere within sincosf's 2 ulp."""
    b = se.recurrence_band_bounds(L=20)
    assert b.shape == (20,) and float(b.max()) <= 1.7e-5, b


@pytest.mark.parametrize("n_p,n_v", [(39, 15), (123, 63), (3, 3)], ids=["one-block P", "two-block P", "none"])
@pytest.mark.parametrize("shape", [(8, 256, 4), (6, 128, 3), (4, 128, -1)], ids=lambda s: "x".join(map(str, s)))
def test_exact_shading_nets_for_other_encodings(shape, n_p, n_v):
    """exact_shading_net's own checks pass (every accumulation exact in any order) for one- and two-block P."""
    sd, x = exact_shading_net(shape, n_p, n_v, rows=512, calib_rows=512)
    assert sd["pts_linears.0.weight"].shape[1] == n_p and x.shape[1] == n_p + n_v
    assert so.shading_shape(sd, n_p) == shape
    assert mlp1_emulate(x, sd, n_p).shape == (512, 4)


@pytest.mark.parametrize("shape", [(6, 128, 3), (4, 256, -1)], ids=lambda s: "x".join(map(str, s)))
def test_emulation_reduces_to_the_10_4_emulation(shape):
    """At 63 + 27 columns mlp1_emulate is shape_emulation.mlp1_emulate, bit for bit."""
    from oracle import shape_emulation as she
    sd, x = she.exact_shading_net(shape, rows=512)
    assert torch.equal(mlp1_emulate(x, sd, 63), she.mlp1_emulate(x, sd))


@pytest.mark.parametrize("L", [0, 6, 16, 20])
def test_posenc_emulation_matches_the_oracle(L):
    v = np.random.default_rng(L).uniform(-1.5, 1.5, (4096, 3)).astype(np.float32)
    emu = se.posenc3(v, L)
    ref = orc.posenc(torch.from_numpy(v).double(), L).numpy()
    bound = np.concatenate([[0.0] * 3] + [[x] * 6 for x in se.recurrence_band_bounds(L=max(L, 1))[:L]])
    assert emu.shape == ref.shape == (4096, 3 + 6 * L)
    assert np.all(np.abs(emu - ref) <= bound + 1e-7 * (1 + np.abs(ref)))


@pytest.mark.parametrize("name,fields,shape", CASES, ids=[c[0] for c in CASES])
def test_oracle_composition_runs_each_case(name, fields, shape):
    scene = case_scene(fields)
    sd0, sd1 = case_weights(scene, shape)
    dirs = torch.from_numpy(se.pixel_dir(64, 64, scene["fov"])[::7].copy())
    out = oracle_render(torch.zeros(3), torch.eye(3), dirs, sd0, sd1, scene, 0.2, 8, return_stages=True)
    n0, n_p, n_v = columns(scene)
    assert out["x0"].shape[1] == n0 and out["x1"].shape[1] == n_p + n_v
    assert torch.isfinite(out["rgb"]).all() and int(out["n_samples"].min()) >= 1


# ------------------------------------------------------------------------------------------------ host surface
@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    from adanerf_b200 import load_library
    return load_library()


def _probe(lib, path):
    from adanerf_b200._lib import Scene
    sc, thr, k, nt = Scene(), C.c_float(), C.c_int(), (C.c_int * 2)()
    return lib.adn_probe_export_dir(str(path).encode(), C.byref(sc), C.byref(thr), C.byref(k), nt), sc


@pytest.mark.parametrize("fields,want,pos_enc,args", [
    (dict(n_freq_pos=-1, n_freq_dir=-1, n_freq_pos0=-1, n_freq_dir0=-1), (-1, -1, -1, -1), "[none, none]", "[10-4, 10-4]"),
    (dict(n_freq_pos=20, n_freq_dir=10, n_freq_pos0=16, n_freq_dir0=4), (20, 10, 16, 4), "[nerf, nerf]", "[16-4, 20-10]"),
    (dict(n_freq_pos=20, n_freq_dir=10, n_freq_pos0=-1, n_freq_dir0=-1), (20, 10, -1, -1), "[none, nerf]", "[10-4, 20-10]"),
])
def test_export_dir_round_trip(lib, tmp_path, fields, want, pos_enc, args):
    from adanerf_b200 import onnx_weights as ow
    scene = dict(orc.SCENE_PAVILLON, **fields)
    sd0, sd1 = case_weights(scene, (6, 128, 3))
    ow.write_export_dir(tmp_path, scene, sd0, sd1, 0.2, 8)
    cfg = (tmp_path / "config.ini").read_text()
    assert f"posEnc = {pos_enc}\n" in cfg and f"posEncArgs = {args}\n" in cfg
    assert "skips = [, 3]" in cfg     # the skip consumer reads W + P columns
    st, sc = _probe(lib, tmp_path)
    assert st == 0 and (sc.n_freq_pos, sc.n_freq_dir, sc.n_freq_pos0, sc.n_freq_dir0) == want


def test_convert_writes_the_encoding(lib, tmp_path):
    from adanerf_b200 import convert
    scene = dict(orc.SCENE_PAVILLON, n_freq_pos=20, n_freq_dir=10, n_freq_pos0=16, n_freq_dir0=4)
    sd0, sd1 = case_weights(scene, (8, 256, 4))
    torch.save(sd0, tmp_path / "n0.weights")
    torch.save(sd1, tmp_path / "n1.weights")
    (tmp_path / "info.txt").write_text("".join(f"{k} = {scene[k]}\n" for k in ("view_cell_center", "view_cell_size", "depth_range",
                                                                              "fov", "max_depth")))
    argv = ["--weights0", str(tmp_path / "n0.weights"), "--weights1", str(tmp_path / "n1.weights"), "--dataset-info",
            str(tmp_path / "info.txt"), "--threshold", "0.2", "--samples", "8", "--out", str(tmp_path / "out")]
    convert.main(argv + ["--pos-enc", "nerf,nerf", "--pos-enc-args", "16-4,20-10"])
    st, sc = _probe(lib, tmp_path / "out")
    assert st == 0 and (sc.n_freq_pos, sc.n_freq_dir, sc.n_freq_pos0, sc.n_freq_dir0) == (20, 10, 16, 4)
    with pytest.raises(ValueError, match="pts_linears.0.weight reads 123 columns, expected 63"):
        convert.main(argv + ["--pos-enc-args", "16-4,10-4"])


@pytest.mark.parametrize("args", ["[10-4, 21-4]", "[10-4, 10-11]", "[16-5, 10-4]"])
def test_loader_rejects_encodings_outside_the_tile_formats(lib, tmp_path, args, capfd):
    from adanerf_b200 import onnx_weights as ow
    sd0, sd1 = orc.make_weights("rand")
    ow.write_export_dir(tmp_path, orc.SCENE_PAVILLON, sd0, sd1, 0.2, 8)
    cfg = (tmp_path / "config.ini").read_text().replace("posEncArgs = [10-4, 10-4]", f"posEncArgs = {args}")
    (tmp_path / "config.ini").write_text(cfg)
    st, _ = _probe(lib, tmp_path)
    assert st == 5   # ADN_ERR_IO
    assert "posEncArgs" in capfd.readouterr().err


def test_check_state_dicts_with_an_encoding():
    from adanerf_b200.convert import check_state_dicts, parse_encoding
    enc = parse_encoding(("nerf", "nerf"), ("16-4", "20-10"))
    assert enc == ((16, 4), (20, 10))
    assert parse_encoding(("none", "nerf"), ("10-4", "6-2")) == ((-1, -1), (6, 2))
    with pytest.raises(ValueError, match="posEncArgs"):
        parse_encoding(("nerf", "nerf"), ("10-4", "21-4"))
    scene = dict(orc.SCENE_PAVILLON, n_freq_pos=20, n_freq_dir=10, n_freq_pos0=16, n_freq_dir0=4)
    sd0, sd1 = case_weights(scene, (8, 256, 4))
    assert check_state_dicts(sd0, sd1, enc) == ((8, 256, -1), (8, 256, 4))
    bad = dict(sd1, **{"views_linears.0.weight": torch.zeros(128, 256 + 27)})
    with pytest.raises(ValueError, match=r"views_linears.0.weight is \[128, 283\], expected \[128, 319\]"):
        check_state_dicts(sd0, bad, enc)
    with pytest.raises(ValueError, match="layers.0.weight reads 126 columns, expected 90"):
        check_state_dicts(sd0, sd1, ((10, 4), (20, 10)))
    with pytest.raises(ValueError):   # without an encoding: today's 10-4 / 2-2 check
        check_state_dicts(sd0, sd1)


@pytest.mark.parametrize("name,fields,shape", CASES, ids=[c[0] for c in CASES])
def test_adapter_reads_the_feature_sets_encodings(name, fields, shape):
    from adanerf_b200.adapter import B200Inference
    from adanerf_b200.renderer import make_scene, scene_columns
    (p0, d0), (p, d) = bands(case_scene(fields))
    none0 = fields.get("n_freq_pos0") == -1
    none1 = fields.get("n_freq_pos") == -1
    fs = lambda none, a, b: SimpleNamespace(enc_type="none" if none else "nerf", n_freq_pos=-1 if none else a,
                                            n_freq_dir=-1 if none else b)
    f0 = fs(none0, p0, d0)
    f1 = fs(none1, p, d)
    f1.__dict__.update(depth_range=[0.1, 8.0], max_depth=8.0, z_near=0.001, z_far=1.0, z_sampler=SimpleNamespace(threshold=0.2),
                       n_ray_samples=8, useNDC=bool(fields.get("use_ndc")), w=800, h=800)
    view = SimpleNamespace(view_cell_center=[0, 0, 0], view_cell_size=[1, 1, 1], fov=1.0, focal=400.0)
    tc = SimpleNamespace(f_in=[f0, f1], dataset_info=SimpleNamespace(view=view), models=[None, None])
    scene, _, _, _ = B200Inference.args_from_train_config(tc)
    assert scene_columns(make_scene(**scene)) == columns(case_scene(fields))


# ------------------------------------------------------------------------------------ against the reference itself
import os  # noqa: E402

from conftest import load_golden  # noqa: E402
from oracle import gen_encoding_golden as geg  # noqa: E402

REFERENCE = os.path.isdir("/root/reference/src")


def _oracle_stages(name, g, sd0, sd1):
    m = g["meta"]
    return oracle_render(torch.from_numpy(g["pose"]), torch.from_numpy(g["rot"]), torch.from_numpy(g["dirs"]), sd0, sd1,
                         m["scene_params"], m["thr"], m["K"], return_stages=True)


def _check_against_reference(name, ref, o, K):
    """The oracle's stages against the reference's: features, raw0, the selection bit for bit from the reference's raw0,
    and rgb / weights on the rays whose sample counts agree."""
    np.testing.assert_allclose(o["x0"].numpy(), ref["x0"], rtol=0, atol=2e-5)
    np.testing.assert_allclose(o["raw0"].numpy(), ref["raw0"], rtol=0, atol=5e-4)
    scene = geg.case_scene(name)
    s2 = orc.stage2_sample(torch.from_numpy(ref["raw0"]), geg.CASES[name][5], K, scene["depth_range"],
                           no_depth_range=bool(scene.get("use_ndc")))
    z = s2["z"].numpy().copy()
    z[~np.isfinite(z)] = np.nan
    np.testing.assert_array_equal(z, ref["z_nan"])
    # stage 3 of the first rays: the reference's [N, K, F] NaN-padded features against the oracle's packed rows
    x1 = ref["x1_nan"]
    live = np.isfinite(x1[..., 0])
    ox1 = o["x1"].numpy()[:int(live.sum())]
    np.testing.assert_allclose(ox1, x1[live], rtol=0, atol=5e-4)
    same = (o["n_samples"].numpy() == np.round(ref["asp"] * K).astype(np.int64))
    assert same.mean() > 0.98
    assert orc.psnr(o["rgb"].numpy()[same], ref["rgb"][same]) > 60.0


@pytest.mark.parametrize("name", list(geg.CASES))
def test_oracle_matches_encoding_golden(name):
    g = load_golden(name)
    sd0, sd1 = geg.case_weights(name)
    o = _oracle_stages(name, g, sd0, sd1)
    n0, n_p, n_v = columns(g["meta"]["scene_params"])
    assert g["x0"].shape[1] == n0 and g["x1_nan"].shape[2] == n_p + n_v
    _check_against_reference(name, g, o, g["meta"]["K"])


@pytest.mark.skipif(not REFERENCE, reason="the reference checkout is not present")
@pytest.mark.parametrize("name", list(geg.CASES))
def test_oracle_matches_live_reference_on_a_fresh_seed(name):
    sd0, sd1 = geg.case_weights(name, seed=5)
    pix, dirs, pose, rot = geg.case_rays(name, n_rays=64, stride=9973)
    r = geg.RefRenderer(name)
    r.load_state_dicts(sd0, sd1)
    ref = r.stages(pose, rot, dirs)
    K = geg.CASES[name][4]
    o = oracle_render(pose, rot, dirs, sd0, sd1, geg.case_scene(name), geg.CASES[name][5], K, return_stages=True)
    ref["x1_nan"] = ref["x1_nan"][:16]
    _check_against_reference(name, ref, o, K)


@pytest.mark.skipif(not REFERENCE, reason="the reference checkout is not present")
@pytest.mark.parametrize("name", list(geg.CASES))
def test_adapter_against_the_live_reference(name):
    """args_from_train_config on the reference's own initialised feature sets gives the case's scene encoding, and a
    renderer scene whose column counts are the reference models' input widths."""
    from adanerf_b200.adapter import B200Inference
    from adanerf_b200.renderer import make_scene, scene_columns
    r = geg.RefRenderer(name)
    scene, models, _, _ = B200Inference.args_from_train_config(r.tc)
    want = geg.case_scene(name)
    for k in ("n_freq_pos", "n_freq_dir", "n_freq_pos0", "n_freq_dir0"):
        assert scene[k] == want[k], (k, scene[k], want[k])
    n0, n_p, n_v = scene_columns(make_scene(**scene))
    sd0, sd1 = models[0].state_dict(), models[1].state_dict()
    assert sd0["layers.0.weight"].shape[1] == n0
    assert sd1["pts_linears.0.weight"].shape[1] == n_p and sd1["views_linears.0.weight"].shape[1] == sd1["alpha_linear.weight"].shape[1] + n_v


@pytest.mark.parametrize("p0,d0,args", [(-1, 4, "[0-4, 10-4]"), (16, -1, "[16-0, 10-4]")])
def test_zero_sampling_band_count_round_trips(lib, tmp_path, p0, d0, args):
    """A sampling encoding with one zero count (nerf 0-4) is written as 0-4 and read back as -1 (zero bands), not as 0
    ("the shading net's count"), so the export's 30-column sampling net matches the scene it loads."""
    from adanerf_b200 import onnx_weights as ow
    from adanerf_b200.renderer import make_scene, scene_columns
    scene = dict(orc.SCENE_PAVILLON, n_freq_pos0=p0, n_freq_dir0=d0)
    torch.manual_seed(0)
    sd0 = orc.init_sampling_net(n_in=columns(scene)[0])
    sd1 = orc.init_shading_net()
    ow.write_export_dir(tmp_path, scene, sd0, sd1, 0.2, 8)
    assert f"posEncArgs = {args}\n" in (tmp_path / "config.ini").read_text()
    st, sc = _probe(lib, tmp_path)
    assert st == 0 and (sc.n_freq_pos0, sc.n_freq_dir0) == (p0, d0)
    assert scene_columns(sc)[0] == sd0["layers.0.weight"].shape[1] == 6 + 6 * max(p0, d0)
