"""The fixed-K sampler (option "sampler" = 1) bit for bit: pdf_sample_kernel and the density composite
(stage5_thread_kernel<true> / stage5_warp_kernel<true>) against the fp32-faithful emulation of oracle/stage_emulation.py,
on whole 800x800 frames of two sampling nets, on edge rows and on synthetic composite inputs; one render_rays frame
against the emulation chain; and deliberately wrong emulations that must differ from the device (teeth).

The emulation takes CUDA's expf and double pow as callables.  Here they are torch's own CUDA kernels (torch.exp /
torch.sigmoid on float32, torch.pow on float64 with a full-tensor base); both sides are CUDA's math library without
fast-math, and test_torch_transcendentals_are_the_kernels checks that they give the kernels' bits before anything
relies on it.  Every comparison is assert_array_equal on int32 views, NaN compared by position (canonical bits)."""
import os
import time

import numpy as np
import pytest
import torch

from adanerf_b200.synthetic import load_weights_npz
from oracle import adanerf_oracle as orc
from oracle import donerf_oracle as dno
from oracle import stage_emulation as se
from test_composite_outputs_exact import _check_epilogue
from test_stage_emulation import _pdf_edge_rows

pytestmark = pytest.mark.gpu

F32, F64 = np.float32, np.float64
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
KS_SAMPLER = [1, 2, 3, 7, 8, 15, 16, 31, 32, 33, 48, 63, 64, 127, 128]
KS_COMPOSITE = [1, 2, 3, 5, 31, 32, 33, 64, 100, 128]
CHUNK = 1 << 17                   # rays per emulation / stage-3 chunk (memory only: every stage is per ray)
BIG_K = 33                        # from here on the emulation checks every 4th ray of the device's whole-frame call
T_START = time.perf_counter()


# ------------------------------------------------------------------------------------ CUDA's transcendentals via torch
def _cuda(a, dtype=F32):
    return torch.from_numpy(np.ascontiguousarray(a, dtype)).cuda()


def expf_cuda(x):
    x = np.asarray(x, F32)
    return torch.exp(_cuda(x)).cpu().numpy() if x.size else x.copy()


def sigmoid_cuda(x):
    x = np.asarray(x, F32)
    return torch.sigmoid(_cuda(x)).cpu().numpy() if x.size else x.copy()


def pow64_cuda(base, x):
    x = np.asarray(x, F32)
    if not x.size:
        return x.astype(F64)
    xx = _cuda(x, F64)
    return torch.pow(torch.full_like(xx, base), xx).cpu().numpy()


def powf_cuda(base, x):
    """fp32 pow on the fp32 base (a tooth)."""
    xx = _cuda(x, F32)
    return torch.pow(torch.full_like(xx, float(F32(base))), xx).cpu().numpy()


def expf_f64(x):
    """Correctly rounded expf through float64 (a tooth: not CUDA's expf)."""
    with np.errstate(over="ignore"):
        return np.exp(np.asarray(x, F32).astype(F64)).astype(F32)


def _bits(a):
    a = np.array(a, F32)
    a[np.isnan(a)] = se.NAN32
    return a.view(np.int32)


def _equal(got, want, what):
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    np.testing.assert_array_equal(_bits(got), _bits(want), err_msg=what)


def _differs(a, b):
    return not np.array_equal(_bits(a), _bits(b))


# ---------------------------------------------------------------------------------------------------------- (a), (b)
def test_torch_transcendentals_are_the_kernels():
    """(a) torch.sigmoid on float32 CUDA tensors, and 1 / (1 + torch.exp(-x)) composed in fp32, equal the library's
    sigmoidf_acc bit for bit: read back as the alpha of the adaptive composite with zp = 1 (alpha = sigmoidf_acc(a) * 1),
    on 16 M logits over [-110, 110], 2 M over the subnormal-result range [-104.5, -86.5], and +-0, +-inf, NaN.
    (b) torch.exp equals the kernel's expf on y in [-ln 2, 0]: 1 - alpha of the density composite at K = 2, z = (0, 1),
    ray_d = (1, 0, 0), density -y, is expf(y) exactly there (Sterbenz)."""
    from adanerf_b200 import Renderer
    r = Renderer(orc.SCENE_PAVILLON)
    rng = np.random.default_rng(0)
    special = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 88.7, -88.7, 103.9, -103.9, 104.0, -104.0], F32)
    x = np.concatenate([rng.uniform(-110, 110, 1 << 24), rng.uniform(-104.5, -86.5, 1 << 21)]).astype(F32)
    x = np.concatenate([special, x, np.zeros((-(x.size + special.size)) % 32, F32)])
    K, n = 32, x.size // 32
    raw1 = np.zeros((x.size, 4), F32)
    raw1[:, 3] = x
    ones = torch.ones(x.size, device="cuda")
    lay = torch.arange(n, dtype=torch.int32, device="cuda")
    kern = r.stage5(_cuda(raw1), ones, ones, lay * K, torch.full_like(lay, K), K, aux=("alpha",))["alpha"].reshape(-1).cpu().numpy()
    a_sig = sigmoid_cuda(x)
    a_exp = F32(1) / (F32(1) + expf_cuda(-x))
    n_sig, n_exp = int((_bits(a_sig) != _bits(kern)).sum()), int((_bits(a_exp) != _bits(kern)).sum())
    print(f"(a) sigmoid: {x.size} logits, torch.sigmoid differs from sigmoidf_acc on {n_sig}, 1 / (1 + torch.exp(-x)) on {n_exp}")

    y = np.concatenate([rng.uniform(-0.6931471, 0.0, 1 << 24), -(10.0 ** rng.uniform(-45, 0, 1 << 20)),
                        [0.0, -0.0, -0.6931471, -2.0 ** -149, -2.0 ** -126, -2.0 ** -24]])
    y = np.clip(y, -0.6931471, 0.0).astype(F32)
    m = y.size
    raw1 = np.zeros((m, 2, 4), F32)
    raw1[:, 0, 3] = -y
    z = np.tile(np.array([0.0, 1.0], F32), m)
    rd = np.tile(np.array([[1.0, 0.0, 0.0]], F32), (m, 1))
    alpha = r.stage5_density(_cuda(raw1.reshape(-1, 4)), _cuda(z), _cuda(rd), 2, aux=("alpha",))["alpha"][:, 0].cpu().numpy()
    n_b = int((_bits(F32(1) - alpha) != _bits(expf_cuda(y))).sum())
    print(f"(b) expf: {m} arguments in [-ln 2, 0], torch.exp differs from the kernel's expf on {n_b}")
    r.close()
    assert n_sig == 0 and n_exp == 0, "(a) torch's CUDA sigmoid / exp is not the kernels' sigmoidf_acc"
    assert n_b == 0, "(b) torch's CUDA exp is not the kernels' expf"


# ------------------------------------------------------------------------------------------------------ frames
def _renderer(nets):
    from adanerf_b200 import Renderer
    if nets == "pav":
        sd0, sd1 = load_weights_npz(os.path.join(GOLDEN, "weights_pavillon"))
        scene = orc.SCENE_PAVILLON
    else:
        sd0, sd1 = orc.make_weights("rand", seed=100)
        scene = orc.SCENE_BARBERSHOP
    r = Renderer(scene, sampling_net=sd0, shading_net=sd1)
    r.set_option("sampler", 1)
    return r, scene


@pytest.fixture(scope="module")
def frames():
    """Per net: the renderer, and stage 0 + the sampling MLP of an 800x800 frame from the view-cell centre (device raw0)."""
    out = {}
    for nets in ("pav", "rand"):
        r, scene = _renderer(nets)
        dirs = r.generate_ray_directions(800, 800)
        pose = torch.tensor(scene["view_cell_center"], dtype=torch.float32)
        x0, ro, rd = r.stage0(pose, torch.eye(3), dirs)
        raw0 = r.mlp0(x0)
        del x0
        out[nets] = dict(r=r, scene=scene, dirs=dirs, pose=pose, ro=ro, rd=rd, raw0=raw0, raw0_h=raw0.cpu().numpy(), cdf={})
    yield out
    for f in out.values():
        f["r"].close()


def _cdf(f, transform):
    """The emulation's staged cdf of the whole frame (it does not depend on K)."""
    if transform not in f["cdf"]:
        raw = f["raw0_h"]
        f["cdf"][transform] = np.concatenate([se.pdf_cdf(se.pdf_transform(raw[i:i + CHUNK], transform, expf_cuda))
                                              for i in range(0, raw.shape[0], CHUNK)])
    return f["cdf"][transform]


def _place(cdf, K, scene, pow64=pow64_cuda, **teeth):
    return np.concatenate([se.pdf_place(cdf[i:i + CHUNK], K, scene, pow64, **teeth) for i in range(0, cdf.shape[0], CHUNK)])


@pytest.mark.parametrize("nets", ["pav", "rand"])
def test_sampler_frame(frames, nets):
    """z of whole 800x800 frames, both transforms, K = 1 ... 128: K + 1 dividing 128 puts u exactly on cdf entries of
    uniform rows, the others run the j = 1 + lane, 33 + lane, ... loop tails.  Every ray up to K = 32, every 4th ray of
    the frame above (the emulation's time grows with K)."""
    f = frames[nets]
    r, scene = f["r"], f["scene"]
    n = f["raw0"].shape[0]
    t0 = time.perf_counter()
    for transform in (dno.SIGMOID, dno.SOFTMAX):
        cdf = _cdf(f, transform)
        for K in KS_SAMPLER:
            s = r.pdf_sample(f["raw0"], K, transform)
            z = s["z"].reshape(n, K).cpu().numpy()
            rows = slice(None, None, 4 if K >= BIG_K else 1)
            _equal(z[rows], _place(cdf[rows], K, scene), f"{nets} transform {transform} K={K}")
            assert (np.diff(z, axis=1) >= 0).all()
            if K in (1, 33, 128):
                assert torch.equal(s["count"].cpu(), torch.full((n,), K, dtype=torch.int32))
                assert torch.equal(s["offset"].cpu(), torch.arange(n, dtype=torch.int32) * K)
                assert torch.equal(s["ray"].cpu(), torch.arange(n, dtype=torch.int32).repeat_interleave(K))
    print(f"{nets}: {n} rays x {len(KS_SAMPLER)} K x 2 transforms bit for bit ({time.perf_counter() - t0:.1f} s)")


def test_sampler_edge_rows(frames):
    """Constant, one-hot, two-spike (clamped runs between, spikes in cells 0 and 127), all -200, subnormal and zero exp,
    +-1e30, -0.0, +-inf and NaN rows through adn_pdf_sample.  A non-finite row's NaN stays in its own ray, at the
    positions the oracle puts it.  Then ray counts 0, 1, 7, 8, 9, 1073 and a raw0 view 4 bytes off 16-byte alignment."""
    f = frames["pav"]
    r, scene = f["r"], f["scene"]
    raw = _pdf_edge_rows()
    finite = np.isfinite(raw).all(1)
    for transform in (dno.SIGMOID, dno.SOFTMAX):
        cdf = se.pdf_cdf(se.pdf_transform(raw, transform, expf_cuda))
        for K in KS_SAMPLER:
            z = r.pdf_sample(_cuda(raw), K, transform)["z"].reshape(-1, K).cpu().numpy()
            _equal(z, se.pdf_place(cdf, K, scene, pow64_cuda), f"edge rows transform {transform} K={K}")
            ref = dno.pdf_sample(torch.from_numpy(raw), K, transform, scene["depth_range"]).numpy()
            np.testing.assert_array_equal(np.isnan(z), np.isnan(ref), err_msg=f"NaN positions transform {transform} K={K}")
            assert not np.isnan(z[finite]).any()
    raw0 = f["raw0"][:1073].contiguous()
    for transform, K in ((dno.SIGMOID, 5), (dno.SOFTMAX, 40)):
        cdf = se.pdf_cdf(se.pdf_transform(raw0.cpu().numpy(), transform, expf_cuda))
        for n in (0, 1, 7, 8, 9, 1073):
            s = r.pdf_sample(raw0[:n], K, transform)
            assert s["z"].numel() == n * K and s["ray"].numel() == n * K
            _equal(s["z"].reshape(n, K).cpu().numpy(), se.pdf_place(cdf[:n], K, scene, pow64_cuda), f"{n} rays K={K}")
            np.testing.assert_array_equal(s["ray"].cpu().numpy(), np.repeat(np.arange(n, dtype=np.int32), K))
            np.testing.assert_array_equal(s["count"].cpu().numpy(), np.full(n, K, np.int32))
            np.testing.assert_array_equal(s["offset"].cpu().numpy(), np.arange(n, dtype=np.int32) * K)
        buf = torch.empty(1073 * 128 + 1, device="cuda")
        buf[1:] = raw0.reshape(-1)
        view = buf[1:].view(1073, 128)
        assert view.data_ptr() % 16 == 4
        _equal(r.pdf_sample(view, K, transform)["z"].cpu().numpy(), r.pdf_sample(raw0, K, transform)["z"].cpu().numpy(),
               f"unaligned raw0 K={K}")


# -------------------------------------------------------------------------------------------------- density composite
def _raw1(r, ro, rd, z, K):
    """Stage 3 then the shading MLP on K samples per ray (z [N K] device), in ray chunks."""
    n = ro.shape[0]
    out = []
    for i in range(0, n, CHUNK):
        m = min(CHUNK, n - i)
        ray = torch.arange(m, dtype=torch.int32, device="cuda").repeat_interleave(K)
        out.append(r.mlp1(r.stage3(ro[i:i + m], rd[i:i + m], ray, z[i * K:(i + m) * K])))
    return torch.cat(out)


def _composite_emu(raw1, z, rd, K):
    """The emulation's density composite in ray chunks: sigmoids from torch, alpha from density_alpha."""
    n = rd.shape[0]
    parts = []
    for i in range(0, n, CHUNK):
        m = min(CHUNK, n - i)
        q = raw1[i * K:(i + m) * K]
        zz = z[i * K:(i + m) * K]
        alpha = se.density_alpha(q[:, 3], zz, rd[i:i + m], K, expf_cuda)
        parts.append(se.stage5_density(sigmoid_cuda(q[:, :3]), alpha, zz, K))
    return {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}


def _check_composite(out, emu, scene, what):
    o = {k: v.cpu().numpy() for k, v in out.items() if v is not None}
    for k in ("rgb", "weights", "alpha", "z_vals", "depth_map", "acc_map"):
        _equal(o[k], emu[k], f"{what}: {k}")
    _check_epilogue(o, scene, what)
    _equal(o["disp_map"], se.disp_map(emu["depth_map"], emu["acc_map"]), f"{what}: disp_map")
    np.testing.assert_array_equal(o["rgba8"], se.rgba8(emu["rgb"]), err_msg=f"{what}: rgba8")


@pytest.mark.parametrize("nets,transform", [("pav", dno.SIGMOID), ("rand", dno.SOFTMAX)])
def test_density_composite_frame(frames, nets, transform):
    """Every output of the density composite on the device's own z and raw1 of a whole frame (stage 3, then the shading
    MLP), K covering both kernels, the 4-wide unroll tails and partial 32-blocks: every ray up to K = 32, every 4th ray
    of the frame above."""
    f = frames[nets]
    r, scene, rd = f["r"], f["scene"], f["rd"]
    rd_h = rd.cpu().numpy()
    t0 = time.perf_counter()
    for K in KS_COMPOSITE:
        z = r.pdf_sample(f["raw0"], K, transform)["z"]
        raw1 = _raw1(r, f["ro"], rd, z, K)
        out = r.stage5_density(raw1, z, rd, K, rgba8=True)
        st = 4 if K >= BIG_K else 1                 # every output's first dimension is the ray
        out = {k: v[::st] for k, v in out.items() if v is not None}
        raw1, z = raw1.reshape(-1, K, 4)[::st].reshape(-1, 4), z.reshape(-1, K)[::st].reshape(-1)
        _check_composite(out, _composite_emu(raw1.cpu().numpy(), z.cpu().numpy(), rd_h[::st], K), scene, f"{nets} K={K}")
    print(f"{nets}: density composite of {rd.shape[0]} rays x {len(KS_COMPOSITE)} K bit for bit ({time.perf_counter() - t0:.1f} s)")


def _synthetic(K, rng, n=1500):
    """raw1 [n K, 4], z [n K], ray_d [n, 3]: negative, NaN and +inf densities, repeated z (dist 0: 0 * inf), decreasing z
    (negative dist: alpha < 0), ray_d of norm 0 and != 1, and rays whose every alpha is 0."""
    raw1 = (rng.standard_normal((n, K, 4)) * 3).astype(F32)
    z = np.sort(rng.uniform(0.2, 8.0, (n, K)), axis=1).astype(F32)
    rd = (rng.standard_normal((n, 3)) * rng.uniform(0.3, 3.0, (n, 1))).astype(F32)
    rd[::50] = 0.0                                             # norm 0
    rd[1::50] = orc.generate_ray_directions(8, 8, 1.0).reshape(-1, 3)[:len(rd[1::50])]   # unit
    raw1[2::10, :, 3] = -np.abs(raw1[2::10, :, 3])             # every alpha 0
    raw1[3::10, :, 3] = np.where(rng.random((len(raw1[3::10]), K)) < 0.2, np.nan, raw1[3::10, :, 3])
    raw1[4::10, :, 3] = np.where(rng.random((len(raw1[4::10]), K)) < 0.2, np.inf, raw1[4::10, :, 3])
    raw1[5::10, rng.integers(K), 3] = np.inf
    z[5::10] = np.repeat(z[5::10, :1], K, 1)                   # repeated z with an inf density: 0 * inf
    z[6::10] = z[6::10, ::-1]                                  # decreasing z: alpha < 0
    z[7::10, K // 2:] = z[7::10, K // 2:K // 2 + 1]            # a repeated tail
    raw1[8::10, :, :3] = np.where(rng.random((len(raw1[8::10]), K, 3)) < 0.1, np.nan, raw1[8::10, :, :3])
    raw1[9::10, :, 3] *= 100.0                                 # alpha = 1 and T underflow
    return raw1.reshape(-1, 4), z.reshape(-1), rd


@pytest.mark.parametrize("K", KS_COMPOSITE)
def test_density_composite_synthetic(frames, K):
    f = frames["rand"]
    r, scene = f["r"], f["scene"]
    raw1, z, rd = _synthetic(K, np.random.default_rng(K))
    out = r.stage5_density(_cuda(raw1), _cuda(z), _cuda(rd), K, rgba8=True)
    emu = _composite_emu(raw1, z, rd, K)
    _check_composite(out, emu, scene, f"synthetic K={K}")
    if K > 1:
        a = emu["alpha"]
        assert (a < 0).any() and np.isnan(a).any() and (a == 1).any()
        assert np.isnan(se.disp_map(emu["depth_map"], emu["acc_map"])).any()


# ------------------------------------------------------------------------------------------------------ the driver
@pytest.mark.parametrize("transform,K", [(dno.SIGMOID, 16), (dno.SOFTMAX, 48)])
def test_render_rays_frame_equals_the_emulation_chain(frames, transform, K):
    """render_rays(want_aux) of an 800x800 frame: z from the emulated sampler on the driver's own raw0, raw1 from the
    device on that z, then the emulated composite -- every output bit for bit."""
    f = frames["pav"]
    r, scene = f["r"], f["scene"]
    r.set_option("pdf_transform", transform)
    o = r.render_rays(f["pose"], torch.eye(3), f["dirs"], 0.0, K, want_oracle_weights=True, want_aux=True)
    raw0 = o["oracle_weights"].cpu().numpy()
    z = np.concatenate([se.pdf_sample(raw0[i:i + CHUNK], K, transform, scene, expf_cuda, pow64_cuda)
                        for i in range(0, raw0.shape[0], CHUNK)]).reshape(-1)
    raw1 = _raw1(r, f["ro"], f["rd"], _cuda(z), K).cpu().numpy()
    emu = _composite_emu(raw1, z, f["rd"].cpu().numpy(), K)
    _equal(o["z_vals"].cpu().numpy(), emu["z_vals"], "z_vals")
    for k in ("rgb", "weights", "alpha", "depth_map", "acc_map"):
        _equal(o[k].cpu().numpy(), emu[k], k)
    _equal(o["disp_map"].cpu().numpy(), se.disp_map(emu["depth_map"], emu["acc_map"]), "disp_map")
    v, bound = se.depth_est_f64(emu["depth_map"], scene)
    de = o["depth_est"].cpu().numpy()
    fin = np.isfinite(v)
    assert (np.abs(de[fin].astype(F64) - v[fin]) <= bound[fin]).all()
    assert (o["n_samples"].cpu() == K).all()


# ------------------------------------------------------------------------------------------------------------ teeth
def test_teeth(frames):
    """Each mutated emulation differs from the device on at least one sample: fp32 CDF, fp32 sequential wsum,
    right=False, no clamp, j * step on both halves of linspace, fp32 pow, float64-rounded expf; for the composite a
    sequential product (tree=False) and lane sums added in order (butterfly=False)."""
    rows = [frames[nets]["raw0_h"][::40] for nets in ("pav", "rand")] + [_pdf_edge_rows()]
    raw = np.concatenate(rows)
    r, scene = frames["pav"]["r"], frames["pav"]["scene"]
    teeth = {"fp32 cdf": dict(scan="fp32"), "fp32 wsum": dict(wsum="fp32"), "right=False": dict(right=False),
             "no clamp": dict(clamp=False), "j step linspace": dict(symmetric=False), "fp32 pow": dict(pow64=powf_cuda),
             "float64 expf": dict(expf=expf_f64)}
    bit = {k: 0 for k in teeth}
    for transform in (dno.SIGMOID, dno.SOFTMAX):
        for K in (7, 33, 128):
            z = r.pdf_sample(_cuda(raw), K, transform)["z"].reshape(-1, K).cpu().numpy()
            _equal(z, se.pdf_sample(raw, K, transform, scene, expf_cuda, pow64_cuda), f"teeth inputs K={K}")
            for name, kw in teeth.items():
                kw = dict(dict(expf=expf_cuda, pow64=pow64_cuda), **kw)
                bad = se.pdf_sample(raw, K, transform, scene, **kw)
                bit[name] += int((_bits(bad) != _bits(z)).sum())
    print("sampler teeth, samples that differ from the device:", bit)
    assert all(v > 0 for v in bit.values()), bit
    f = frames["pav"]
    K, n = 64, 1 << 14
    zd = r.pdf_sample(f["raw0"][:n], K, dno.SIGMOID)["z"]
    raw1 = _raw1(r, f["ro"][:n], f["rd"][:n], zd, K).cpu().numpy()
    out = r.stage5_density(_cuda(raw1), zd, f["rd"][:n], K)
    rd_h, z_h = f["rd"][:n].cpu().numpy(), zd.cpu().numpy()
    alpha = se.density_alpha(raw1[:, 3], z_h, rd_h, K, expf_cuda)
    sig = sigmoid_cuda(raw1[:, :3])
    args = (sig, None, z_h, np.arange(n) * K, np.full(n, K), K)
    _equal(out["weights"].cpu().numpy(), se.stage5_warp(*args, alpha=alpha)["weights"], "teeth composite inputs")
    for kw in (dict(tree=False), dict(butterfly=False)):
        bad = se.stage5_warp(*args, alpha=alpha, **kw)
        assert any(_differs(out[k].cpu().numpy(), bad[k]) for k in ("rgb", "weights", "depth_map", "acc_map")), kw
    print(f"test_donerf_exact_gpu.py: {time.perf_counter() - T_START:.1f} s since import")
