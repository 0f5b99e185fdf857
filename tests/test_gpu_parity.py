"""GPU parity tests: every CUDA stage is driven through the C ABI (ctypes) and compared with the
golden fixtures produced by the unmodified reference and with the CPU oracle on the same inputs.
Tolerances (stated per test) follow SURVEY.md 8(d): integer / index work bit-exact, fp32 SIMT stages
~1e-6 (5e-4 on the 2^9 posenc band), MLPs by their reduced-precision budget, end-to-end by PSNR."""
import numpy as np
import pytest
import torch

from conftest import case_weights, load_golden
from oracle import adanerf_oracle as orc
from oracle import mlp_emulation as me

pytestmark = pytest.mark.gpu

CASES = ["pav_k8_t0.2", "pav_k8_t0.5", "pav_k16_t0.15", "shaped_k8_t0.2", "rand_k8_t0.2"]


def _renderer(scene, sd0=None, sd1=None):
    from adanerf_b200 import Renderer
    return Renderer(scene, device=0, sampling_net=sd0, shading_net=sd1)


@pytest.fixture(scope="module")
def bare():
    r = _renderer(orc.SCENE_BARBERSHOP)
    yield r
    r.close()


def _packed_from_golden(g, K):
    """Packed (ray-major, depth-ascending) views of the NaN/zero padded golden tensors."""
    z = g["z_nan"]
    mask = np.isfinite(z)
    ray = np.repeat(np.arange(z.shape[0]), K).reshape(z.shape)[mask]
    return mask, ray, z[mask]


# ------------------------------------------------------------------------------- wgmma bring-up
# Kernel vs the bf16-faithful emulation (the fp32 accumulation order is all that differs): 2x the values measured on an
# H100 80GB HBM3 -- single layer, max abs err by terms: 7.63e-6 (3), 2.86e-6 (1); multi-layer, max err / output scale by
# depth: 2.7e-6 (2), 6.7e-6 (3), 1.23e-5 (8).  The deeper split nets carry about what fp32 accumulation costs per layer,
# so against fp64 they measure nearly the same.
UMMA_SINGLE_BOUND = {3: 1.6e-5, 1: 6e-6}
UMMA_MULTI_BOUND = {2: 6e-6, 3: 1.4e-5, 8: 2.5e-5}
@pytest.mark.parametrize("n_out", [128, 256])
@pytest.mark.parametrize("terms", [3, 1])
def test_umma_single_layer(bare, n_out, terms):
    """One Linear layer through the wgmma path == validates descriptors, swizzle, accumulator fragment layout.  Compared
    with the bf16-faithful emulation (same operands, float64 sums), so only the fp32 accumulation order differs."""
    g = torch.Generator().manual_seed(5)
    W = torch.randn(n_out, 90, generator=g) * 0.3
    b = torch.randn(n_out, generator=g) * 0.1
    x = torch.randn(300, 90, generator=g)
    sd = {"layers.0.weight": W, "layers.0.bias": b}
    bare.set_option("mlp0_terms", terms)
    bare.set_weights(0, sd)
    out = bare.mlp0(x.cuda(), n_out=n_out)
    emu = me.mlp0_emulate(x.cuda(), sd, terms=terms)
    ref64 = x.double() @ W.double().T + b.double()
    err = (out - emu).abs().max().item()
    err64 = (out.cpu().double() - ref64).abs().max().item()
    print(f"single layer n_out={n_out} terms={terms}: max abs err {err:.3e} vs emulation, {err64:.3e} vs fp64")
    assert err < UMMA_SINGLE_BOUND[terms]
    # bf16x3 keeps ~16 mantissa bits per operand: |err| ~ 2^-16 * |x||w| * sqrt(K)
    assert err64 < (2e-4 if terms == 3 else 6e-2)
    bare.set_option("mlp0_terms", 3)


@pytest.mark.parametrize("depth", [2, 3, 8])
def test_umma_multi_layer(bare, depth):
    g = torch.Generator().manual_seed(depth)
    sd = {}
    dims = [90] + [256] * (depth - 1) + [128]
    for i in range(depth):
        sd[f"layers.{i}.weight"] = torch.randn(dims[i + 1], dims[i], generator=g) * (1.4 / dims[i] ** 0.5)
        sd[f"layers.{i}.bias"] = torch.randn(dims[i + 1], generator=g) * 0.1
    x = torch.randn(1000, 90, generator=g)
    bare.set_weights(0, sd)
    out = bare.mlp0(x.cuda())
    emu = me.mlp0_emulate(x.cuda(), sd, terms=3)
    ref = orc.mlp0_forward(x.double(), orc.to_dtype(sd, torch.float64)).float()
    scale = max(1.0, ref.abs().max().item())
    err = (out - emu).abs().max().item()
    err64 = (out.cpu() - ref).abs().max().item()
    print(f"depth {depth}: max abs err {err:.3e} vs emulation, {err64:.3e} vs fp64 (ref scale {scale:.2f})")
    assert err < UMMA_MULTI_BOUND[depth] * scale
    assert err64 < 1e-4 * scale


# ------------------------------------------------------------------------------------ stage 0
def test_generate_ray_directions_bit_exact(bare):
    W, H = 800, 800
    d = bare.generate_ray_directions(W, H, row0=0, rows=H).cpu().numpy()
    ref = orc.generate_ray_directions(W, H, orc.SCENE_BARBERSHOP["fov"]).reshape(-1, 3).astype(np.float32)
    np.testing.assert_array_equal(d, ref)
    band = bare.generate_ray_directions(W, H, row0=300, rows=7).cpu().numpy()
    np.testing.assert_array_equal(band, ref[300 * W:307 * W])


@pytest.mark.parametrize("W,H,row0,rows", [(1, 1, 0, 1), (3, 801, 400, 1), (801, 799, 798, 1), (1920, 1080, 517, 64)])
def test_generate_ray_directions_frame_sizes(bare, W, H, row0, rows):
    """Other frame sizes (a single pixel, odd and non-square frames, 1080p): the whole frame and the band
    [row0, row0 + rows) (what one tile of a multi-GPU frame generates), bit for bit."""
    d = bare.generate_ray_directions(W, H, row0=0, rows=H).cpu().numpy()
    ref = orc.generate_ray_directions(W, H, orc.SCENE_BARBERSHOP["fov"]).reshape(-1, 3).astype(np.float32)
    np.testing.assert_array_equal(d, ref)
    band = bare.generate_ray_directions(W, H, row0=row0, rows=rows).cpu().numpy()
    np.testing.assert_array_equal(band, ref[row0 * W:(row0 + rows) * W])


@pytest.mark.parametrize("case", CASES)
def test_stage0_matches_reference(case):
    g = load_golden(case)
    r = _renderer(g["meta"]["scene_params"])
    x0, ro, rd = r.stage0(g["pose"], g["rot"], torch.from_numpy(g["dirs"]).cuda())
    np.testing.assert_array_equal(rd.cpu().numpy(), g["ray_d"])                  # FMA chain of ATen bmm
    np.testing.assert_allclose(ro.cpu().numpy(), g["ray_o"], rtol=0, atol=1e-6)
    x0 = x0.cpu().numpy()
    np.testing.assert_allclose(x0[:, :27], g["x0"][:, :27], rtol=0, atol=2e-6)    # direction block
    # position block: frequency 2^k amplifies a 1-ulp position difference by 2^k
    err = np.abs(x0[:, 27:] - g["x0"][:, 27:])
    assert err.max() < 5e-4, err.max()
    assert err[:, :3 + 6 * 4].max() < 2e-5
    r.close()


# ------------------------------------------------------------------------------------ stage 1
@pytest.mark.parametrize("case", ["pav_k8_t0.2", "shaped_k8_t0.2", "rand_k8_t0.2"])
def test_mlp0_matches_reference(case):
    g = load_golden(case)
    sd0, _ = case_weights(case)
    r = _renderer(g["meta"]["scene_params"], sd0=sd0)
    raw0 = r.mlp0(torch.from_numpy(g["x0"]).cuda()).cpu().numpy()
    ref64 = orc.mlp0_forward(torch.from_numpy(g["x0"]).double(), orc.to_dtype(sd0, torch.float64)).numpy()
    scale = max(1.0, np.abs(g["raw0"]).max())
    err_ref = np.abs(raw0 - g["raw0"]).max() / scale
    err64 = np.abs(raw0 - ref64).max() / scale
    noise = np.abs(g["raw0"] - ref64).max() / scale          # the fp32 reference's own distance to fp64
    flips = ((raw0 >= g["meta"]["thr"]) != (g["raw0"] >= g["meta"]["thr"])).mean()
    print(f"{case}: |ours-ref|={err_ref:.2e} |ours-f64|={err64:.2e} |ref-f64|={noise:.2e} threshold flips={flips:.2e}")
    assert err64 < 5e-5, "split-precision sampling MLP must be fp32-class"
    assert flips <= 3.1e-5              # at most one borderline cell of the 256 x 128 (SURVEY.md 8d budget: flips <= 1e-5 .. 3e-5)
    r.close()


# ------------------------------------------------------------------------------------ stage 2
@pytest.mark.parametrize("case", CASES)
def test_stage2_bit_exact_on_reference_raw0(case, bare):
    g = load_golden(case)
    m = g["meta"]
    K = m["K"]
    r = _renderer(m["scene_params"])
    s2 = r.stage2(torch.from_numpy(g["raw0"]).cuda(), m["thr"], K)
    mask, ray, z = _packed_from_golden(g, K)
    cnt = mask.sum(1)
    np.testing.assert_array_equal(s2["count"].cpu().numpy(), cnt)
    np.testing.assert_array_equal(s2["offset"].cpu().numpy(), np.concatenate([[0], np.cumsum(cnt)[:-1]]))
    assert s2["total"] == cnt.sum()
    np.testing.assert_array_equal(s2["ray"].cpu().numpy(), ray)
    # cell ids: invert the golden z through the oracle's cell table
    o2 = orc.stage2_sample(torch.from_numpy(g["raw0"]), m["thr"], K, m["scene_params"]["depth_range"])
    np.testing.assert_array_equal(s2["cell"].cpu().numpy(), o2["cell"].numpy()[mask])
    np.testing.assert_array_equal(s2["zp"].cpu().numpy(), o2["zp"].numpy()[mask])
    np.testing.assert_allclose(s2["z"].cpu().numpy(), z, rtol=2.5e-7, atol=1e-7)   # pow: <= 1-2 ulp
    r.close()


def _stage2_adversarial(n=64 * 5 + 37):
    """Rows built from the values selection can get wrong: -0.0 against +0.0 ties, denormals, +-inf, values equal to a
    threshold and one ulp either side of it; some rows are nothing but one such value.  n is not a multiple of the 64-ray
    tile."""
    rng = np.random.default_rng(12)
    f = np.float32
    t2, t5 = f(0.2), f(0.5)
    special = np.array([0.0, -0.0, 2.0 ** -149, -(2.0 ** -149), 3 * 2.0 ** -149, 2.0 ** -126, 1e-40, np.inf, -np.inf,
                        t2, np.nextafter(t2, f(1)), np.nextafter(t2, f(0)), t5, np.nextafter(t5, f(1)), np.nextafter(t5, f(0)),
                        -t2, 1.0, -1.0], f)
    raw = rng.choice(special, (n, 128))
    mixed = rng.random((n, 128)) < 0.5
    raw[mixed] = rng.uniform(-0.5, 0.7, int(mixed.sum())).astype(f)
    for i, v in enumerate(special):                      # single-valued rows (every cell ties)
        raw[i] = v
    raw[len(special)] = np.where(np.arange(128) % 2 == 0, f(-0.0), f(0.0))
    raw[len(special) + 1] = np.where(np.arange(128) % 3 == 0, f(np.inf), f(-np.inf))
    return torch.from_numpy(raw)


def test_stage2_stress_vectors(bare):
    """Ties, all-equal rows, value == thr, nothing above thr, signed zeros, denormals, infinities ... against the oracle
    (ties lower-cell-first) at every K: <= 8 / <= 16 the two thread-per-ray kernels, above the warp-per-ray kernel.  At
    K <= 16 a raw0 that is only 4-byte aligned (the warp kernel's fallback) gives the same result as the aligned one."""
    g = load_golden("stage2_stress")
    dr = g["meta"]["depth_range"]
    sets = [(torch.from_numpy(g["raw0"]), (0.2, 0.5)), (_stage2_adversarial(), (0.2, 0.5, 3 * 2.0 ** -149))]
    for raw0, thrs in sets:
        n = raw0.shape[0]
        shifted = torch.empty(n * 128 + 1, dtype=torch.float32, device="cuda")[1:].view(n, 128)
        shifted.copy_(raw0)
        assert shifted.data_ptr() % 16 == 4
        for K in range(1, 129):
            for thr in thrs:
                s2 = bare.stage2(raw0.cuda(), thr, K)
                o2 = orc.stage2_sample(raw0, thr, K, dr)
                mask = torch.isfinite(o2["z"]).numpy()
                np.testing.assert_array_equal(s2["count"].cpu().numpy(), o2["count"].numpy(), err_msg=f"K={K} thr={thr}")
                np.testing.assert_array_equal(s2["cell"].cpu().numpy(), o2["cell"].numpy()[mask], err_msg=f"K={K} thr={thr}")
                np.testing.assert_array_equal(s2["zp"].cpu().numpy(), o2["zp"].numpy()[mask], err_msg=f"K={K} thr={thr}")
                if K <= 16:
                    s2m = bare.stage2(shifted, thr, K)
                    for k in ("count", "offset", "cell", "ray", "z", "zp"):
                        assert torch.equal(s2m[k], s2[k]), (K, thr, k)


def test_stage2_large_properties(bare):
    """Full-frame size: offsets are the exclusive scan of counts, packed rays sorted, cells ascending
    inside a ray, deterministic across runs; empty and ragged inputs."""
    g = torch.Generator().manual_seed(3)
    n = 640000
    raw0 = (torch.rand(n, 128, generator=g) * 1.2 - 0.8).cuda()
    a = bare.stage2(raw0, 0.2, 8)
    b = bare.stage2(raw0, 0.2, 8)
    cnt = a["count"].long()
    assert int(cnt.min()) >= 1 and int(cnt.max()) <= 8
    assert torch.equal(a["offset"].long(), torch.cumsum(cnt, 0) - cnt)
    assert a["total"] == int(cnt.sum())
    for k in ("count", "offset", "cell", "ray", "z", "zp"):
        assert torch.equal(a[k], b[k]), k
    ray = a["ray"].long()
    assert bool((ray[1:] >= ray[:-1]).all())
    same = ray[1:] == ray[:-1]
    assert bool((a["cell"][1:][same] > a["cell"][:-1][same]).all())
    vals = raw0[ray, a["cell"].long()]
    assert torch.equal(vals, a["zp"])
    e = bare.stage2(raw0[:0], 0.2, 8)
    assert e["total"] == 0
    one = bare.stage2(raw0[:1], 0.2, 8)
    assert one["total"] == int(one["count"][0])


# ------------------------------------------------------------------------------------ stage 3
@pytest.mark.parametrize("case", ["pav_k8_t0.2", "shaped_k8_t0.2"])
def test_stage3_matches_reference(case):
    g = load_golden(case)
    m = g["meta"]
    K = m["K"]
    r = _renderer(m["scene_params"])
    mask, ray, z = _packed_from_golden(g, K)
    x1 = r.stage3(torch.from_numpy(g["ray_o"]), torch.from_numpy(g["ray_d"]), torch.from_numpy(ray.astype(np.int32)),
                  torch.from_numpy(z)).cpu().numpy()
    ref = g["x1_nan"].reshape(-1, 90)[mask.flatten()]
    err = np.abs(x1 - ref)
    assert err[:, 63:].max() < 2e-6                 # direction block
    assert err[:, :3 + 6 * 4].max() < 2e-5          # low position bands
    assert err.max() < 5e-4, err.max()              # 2^9 band
    r.close()


# ------------------------------------------------------------------------------------ stage 4
@pytest.mark.parametrize("case", ["pav_k8_t0.2", "shaped_k8_t0.2"])
def test_mlp1_matches_reference(case):
    g = load_golden(case)
    m = g["meta"]
    _, sd1 = case_weights(case)
    r = _renderer(m["scene_params"], sd1=sd1)
    mask, _, _ = _packed_from_golden(g, m["K"])
    x1 = g["x1_nan"].reshape(-1, 90)[mask.flatten()]
    raw1 = r.mlp1(torch.from_numpy(x1).cuda()).cpu().numpy()
    ref = g["raw1_pad"].reshape(-1, 4)[mask.flatten()]
    # emulate bf16 operands with fp32 accumulate on the CPU for a like-for-like bound
    err = np.abs(raw1 - ref)
    scale = max(1.0, np.abs(ref).max())
    s_ours = 1 / (1 + np.exp(-raw1.astype(np.float64)))
    s_ref = 1 / (1 + np.exp(-ref.astype(np.float64)))
    p = orc.psnr(s_ours, s_ref)
    print(f"{case}: max|raw1 err|={err.max():.3e} (scale {scale:.2f}) PSNR(sigmoid)={p:.1f} dB")
    assert np.isfinite(raw1).all()
    assert err.max() < 0.05 * scale
    assert p >= 49.4
    r.close()


# ------------------------------------------------------------------------------------ stage 5
@pytest.mark.parametrize("case", CASES)
def test_stage5_matches_reference(case):
    g = load_golden(case)
    m = g["meta"]
    K = m["K"]
    r = _renderer(m["scene_params"])
    mask, ray, z = _packed_from_golden(g, K)
    cnt = mask.sum(1).astype(np.int32)
    off = np.concatenate([[0], np.cumsum(cnt)[:-1]]).astype(np.int32)
    raw1 = g["raw1_pad"].reshape(-1, 4)[mask.flatten()]
    o2 = orc.stage2_sample(torch.from_numpy(g["raw0"]), m["thr"], K, m["scene_params"]["depth_range"])
    zp = o2["zp"].numpy()[mask]
    out = r.stage5(torch.from_numpy(raw1), torch.from_numpy(zp), torch.from_numpy(z), torch.from_numpy(off),
                   torch.from_numpy(cnt), K)
    np.testing.assert_allclose(out["rgb"].cpu().numpy(), g["rgb"], rtol=0, atol=1e-6)
    np.testing.assert_allclose(out["weights"].cpu().numpy(), g["weights"], rtol=0, atol=1e-6)
    r.close()


def test_stage5_dense_warp_path(bare):
    """K > 32 uses the warp-per-ray product scan; compare with the oracle composite."""
    g = torch.Generator().manual_seed(9)
    n, K = 300, 128
    cnt = torch.randint(1, K + 1, (n,), generator=g, dtype=torch.int32)
    off = (torch.cumsum(cnt, 0) - cnt).int()
    M = int(cnt.sum())
    raw1 = torch.randn(M, 4, generator=g)
    zp = torch.rand(M, generator=g) * 0.5
    z = torch.rand(M, generator=g) * 5
    out = bare.stage5(raw1, zp, z, off, cnt, K)
    mapping = (torch.arange(K)[None, :] < cnt[:, None]).flatten()
    zp_pad = torch.zeros(n * K)
    zp_pad[mapping] = zp
    ref = orc.stage5_composite(raw1, z, zp_pad.view(n, K), mapping, n, K)
    np.testing.assert_allclose(out["rgb"].cpu().numpy(), ref["rgb"].numpy(), rtol=0, atol=2e-6)
    np.testing.assert_allclose(out["weights"].cpu().numpy(), ref["weights"].numpy(), rtol=0, atol=2e-6)
    np.testing.assert_allclose(out["depth_map"].cpu().numpy(), ref["depth_map"].numpy(), rtol=0, atol=2e-5)


# ------------------------------------------------------------------------------- end to end
@pytest.mark.parametrize("case", CASES)
def test_render_matches_reference(case):
    g = load_golden(case)
    m = g["meta"]
    sd0, sd1 = case_weights(case)
    r = _renderer(m["scene_params"], sd0, sd1)
    out = r.render_rays(g["pose"], g["rot"], torch.from_numpy(g["dirs"]).cuda(), m["thr"], m["K"], want_oracle_weights=True)
    rgb = out["rgb"].cpu().numpy()
    ns = out["n_samples"].cpu().numpy()
    same = (ns == np.round(g["asp"] * m["K"]).astype(np.int32))
    p = orc.psnr(rgb, g["rgb"])
    print(f"{case}: rays with identical sample count {same.mean():.4f}; PSNR(ours, reference) = {p:.2f} dB")
    assert np.isfinite(rgb).all()
    assert same.mean() >= 0.999         # contract: identical sample count on >= 99.9 % of the rays
    np.testing.assert_allclose(out["oracle_weights"].cpu().numpy(), g["raw0"], rtol=0, atol=2e-4 * max(1, np.abs(g["raw0"]).max()))
    if case.startswith("rand"):
        # untrained nets: alpha*zp leaves [0,1] and amplifies (SURVEY 7c) -> relative check only
        assert np.abs(rgb - g["rgb"]).max() < 0.05 * max(1.0, np.abs(g["rgb"]).max())
    else:
        assert p >= 49.4                # |dPSNR| < 0.05 dB for a 30 dB scene (SURVEY.md 8d)
    host = r.render_rays_host(g["pose"], g["rot"], g["dirs"], m["thr"], m["K"])
    np.testing.assert_array_equal(host["rgb"], rgb)          # host-buffer entry == device entry, bitwise
    np.testing.assert_array_equal(host["n_samples"], ns)
    r.close()


@pytest.mark.parametrize("case", ["pav_k8_t0.2", "pav_k8_t0.5", "shaped_k8_t0.2"])
def test_render_auxiliary_outputs(case):
    """adn_render_rays_aux: weights / alpha / z_vals [N,K], depth / acc / disparity / NeRFOutputDepth [N] against the
    reference's inference dict (golden) and against the oracle on the same per-sample values."""
    g = load_golden(case)
    m = g["meta"]
    K = m["K"]
    sd0, sd1 = case_weights(case)
    r = _renderer(m["scene_params"], sd0, sd1)
    dirs = torch.from_numpy(g["dirs"]).cuda()
    out = r.render_rays(g["pose"], g["rot"], dirs, m["thr"], K, want_aux=True)
    plain = r.render_rays(g["pose"], g["rot"], dirs, m["thr"], K)
    assert torch.equal(out["rgb"], plain["rgb"])                     # asking for more does not change the image
    ns = out["n_samples"].cpu().numpy()
    same = (ns == np.round(g["asp"] * K).astype(np.int32))
    assert same.mean() >= 0.999
    w, a, z = (out[k].cpu().numpy() for k in ("weights", "alpha", "z_vals"))
    # padding exactly like the reference's: zeros / NaN behind the ray's samples
    slot = np.arange(K)[None, :] >= ns[:, None]
    assert (w[slot] == 0).all() and (a[slot] == 0).all() and np.isnan(z[slot]).all() and np.isfinite(z[~slot]).all()
    np.testing.assert_allclose(z[same], g["z_nan"][same], rtol=3e-7, atol=0, equal_nan=True)
    # bf16 shading net: compare like the image (SURVEY 8d), weights / alpha live in [0, 1] for trained / shaped nets
    for name, ours, ref in (("weights", w[same], g["weights"][same]), ("alpha", a[same], g["alpha"][same]),
                            ("depth_est", out["depth_est"].cpu().numpy()[same], g["depth_est"][same, 0])):
        err = np.abs(ours - ref)
        print(f"{case} {name}: max err {err.max():.3e}, mean {err.mean():.3e}")
        assert err.max() < 6e-2 and err.mean() < 3e-3, name
    # internal consistency, exact up to summation order: acc = sum w, depth = sum w z, disparity, log warp
    wt, zt = out["weights"].double(), torch.nan_to_num(out["z_vals"], nan=0.0).double()
    acc, dm = wt.sum(1), (wt * zt).sum(1)
    np.testing.assert_allclose(out["acc_map"].cpu().numpy(), acc.cpu().numpy(), rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(out["depth_map"].cpu().numpy(), dm.cpu().numpy(), rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(out["disp_map"].cpu().numpy(),
                               (1.0 / torch.clamp(out["depth_map"] / out["acc_map"], min=1e-10)).cpu().numpy(), rtol=1e-5)
    de = orc.log_from_world(out["depth_map"].cpu(), m["scene_params"]["depth_range"]).numpy()
    np.testing.assert_allclose(out["depth_est"].cpu().numpy(), de, rtol=0, atol=2e-6)
    only = r.render_rays(g["pose"], g["rot"], dirs, m["thr"], K, want_aux=("depth_est",))
    assert torch.equal(only["depth_est"], out["depth_est"]) and "weights" not in only
    r.close()


def test_render_auxiliary_outputs_chunked_and_dense():
    """Aux buffers are windowed per internal chunk; dense mode (K = 128) goes through the warp-per-ray composite."""
    scene = orc.SCENE_BARBERSHOP
    sd0, sd1 = orc.make_weights("shaped", seed=0)
    r = _renderer(scene, sd0, sd1)
    pose, rot = torch.tensor(scene["view_cell_center"]), torch.eye(3)
    dirs = torch.from_numpy(orc.generate_ray_directions(800, 800, scene["fov"]).reshape(-1, 3)).float()[::97][:6000].cuda()
    one = r.render_rays(pose, rot, dirs, 0.2, 8, want_aux=True)
    r.set_option("chunk_rays", 1024)
    many = r.render_rays(pose, rot, dirs, 0.2, 8, want_aux=True)
    r.set_option("chunk_rays", 0)
    for k in ("rgb",) + r.AUX_KEYS:
        assert torch.equal(torch.nan_to_num(one[k], nan=-1.0), torch.nan_to_num(many[k], nan=-1.0)), k
    d = r.render_rays(pose, rot, dirs[:512], 0.0, 128, want_aux=True)
    ref = orc.render_rays(pose, rot, dirs[:512].cpu(), sd0, sd1, scene, 0.0, 128, return_stages=True)
    assert torch.isfinite(d["z_vals"]).all()
    np.testing.assert_allclose(d["z_vals"].cpu().numpy(), ref["z"].numpy(), rtol=3e-7, atol=5e-7)
    # bf16 shading net on 128 samples per ray; sanity-level bounds (the image-level check is test_render_dense_config1)
    # untrained nets: alpha * zp leaves [0, 1] and the cumprod amplifies (SURVEY 7c) -> relative to the tensor's scale
    for k_ours, k_ref in (("weights", "weights"), ("acc_map", "acc")):
        ours, want = d[k_ours].cpu().numpy(), ref[k_ref].numpy()
        assert np.abs(ours - want).max() < 0.05 * max(1.0, np.abs(want).max()), k_ours
    r.close()


def test_render_dense_config1():
    """BASELINE config 1: first 1024 rays of the 800x800 grid, dense 128 samples, random init."""
    g = load_golden("rand_dense_k128")
    m = g["meta"]
    sd0, sd1 = case_weights("rand_dense_k128")
    r = _renderer(m["scene_params"], sd0, sd1)
    out = r.render_rays(g["pose"], g["rot"], torch.from_numpy(g["dirs"]).cuda(), 0.0, 128, want_oracle_weights=True)
    rgb = out["rgb"].cpu().numpy()
    assert (out["n_samples"].cpu().numpy() == 128).all()
    np.testing.assert_allclose(out["oracle_weights"].cpu().numpy(), g["raw0"], rtol=0, atol=2e-4 * np.abs(g["raw0"]).max())
    scale = max(1.0, np.abs(g["rgb"]).max())
    rel = np.abs(rgb - g["rgb"]).max() / scale
    print(f"dense config 1: max rel err {rel:.3e} (|rgb| scale {scale:.3g})")
    assert np.isfinite(rgb).all()
    assert rel < 0.05
    r.close()


def test_full_frame_properties_and_tiling():
    """800x800 frame through adn_render_camera: deterministic; a row band rendered alone equals the
    same rows of the full frame bit for bit (the multi-GPU tiling invariant); chunked == unchunked."""
    scene = orc.SCENE_BARBERSHOP
    sd0, sd1 = orc.make_weights("shaped", seed=0)
    r = _renderer(scene, sd0, sd1)
    pose = torch.tensor(scene["view_cell_center"])
    rot = torch.eye(3)
    W = H = 800
    full = r.render_camera(pose, rot, W, H, 0.2, 8, want_nsamples=True)
    again = r.render_camera(pose, rot, W, H, 0.2, 8, want_nsamples=True)
    assert torch.equal(full["rgb"], again["rgb"]) and torch.equal(full["n_samples"], again["n_samples"])
    band = r.render_camera(pose, rot, W, H, 0.2, 8, row0=200, rows=100, want_nsamples=True)
    assert torch.equal(band["rgb"], full["rgb"][200 * W:300 * W])
    assert torch.equal(band["n_samples"], full["n_samples"][200 * W:300 * W])
    r.set_option("chunk_rays", 65536)
    chunked = r.render_camera(pose, rot, W, H, 0.2, 8)
    assert torch.equal(chunked["rgb"], full["rgb"])
    r.set_option("chunk_rays", 0)
    st = r.stats()
    assert st["n_samples"] > 0
    # parity on a strided subset of the frame against the oracle
    idx = torch.arange(0, W * H, 4099)
    dirs = torch.from_numpy(orc.generate_ray_directions(W, H, scene["fov"]).reshape(-1, 3)).float()[idx]
    ref = orc.render_rays(pose, rot, dirs, sd0, sd1, scene, 0.2, 8)
    p = orc.psnr(full["rgb"].cpu()[idx], ref["rgb"])
    same = (full["n_samples"].cpu()[idx].long() == ref["n_samples"]).float().mean().item()
    print(f"full frame subset: PSNR {p:.2f} dB, identical counts {same:.4f}, mean spr {full['n_samples'].float().mean():.2f}")
    assert p >= 49.4 and same >= 0.999
    rgba = r.render_camera_rgba8(pose, rot, W, H, 0.2, 8, row0=0, rows=4).cpu()
    expect = (full["rgb"][:4 * W].clamp(0, 1) * 255.0).to(torch.uint8).cpu()
    assert torch.equal(rgba[:, :3], expect) and bool((rgba[:, 3] == 255).all())
    r.close()


def test_error_paths(bare):
    from adanerf_b200 import AdnError
    r = _renderer(orc.SCENE_BARBERSHOP)
    with pytest.raises(AdnError) as e:
        r.render_camera(torch.zeros(3), torch.eye(3), 8, 8, 0.2, 8)
    assert e.value.status == 4          # weights not set
    with pytest.raises(AdnError):
        r.set_weights(1, {"pts_linears.0.weight": torch.zeros(256, 60)})
    sd0, sd1 = orc.make_weights("rand", seed=0)
    r.set_weights(0, sd0)
    r.set_weights(1, sd1)
    with pytest.raises(AdnError):
        r.render_camera(torch.zeros(3), torch.eye(3), 8, 8, 0.0, 8)   # dense needs K == 128
    with pytest.raises(AdnError):
        r.render_camera(torch.zeros(3), torch.eye(3), 8, 8, 0.2, 0)
    r.close()


def _entry_status(r, entry, thr=0.2, K=8, row0=0, rows=8, W=8, H=8):
    """Status of one call of a render entry point straight through the C ABI (the Python wrappers size their outputs from
    the arguments first).  The rays entry points take rows * W rays."""
    import ctypes as C
    from adanerf_b200._lib import AuxOutputs
    n = rows * W
    pose = (C.c_float * 3)(*orc.SCENE_BARBERSHOP["view_cell_center"])
    rot = (C.c_float * 9)(1, 0, 0, 0, 1, 0, 0, 0, 1)
    dirs = torch.from_numpy(orc.generate_ray_directions(W, H, orc.SCENE_BARBERSHOP["fov"]).reshape(-1, 3)).float()
    d_dirs, d_out = dirs.cuda(), torch.empty((W * H, 4), dtype=torch.float32, device="cuda")
    d_ns = torch.empty((W * H,), dtype=torch.int32, device="cuda")
    h_dirs, h_rgb, h_ns = dirs.numpy(), np.empty((W * H, 3), np.float32), np.empty((W * H,), np.int32)
    lib, h = r.lib, r.handle
    calls = {
        "rays": lambda: lib.adn_render_rays(h, pose, rot, d_dirs.data_ptr(), n, thr, K, d_out.data_ptr(), d_ns.data_ptr(), None, None),
        "rays_aux": lambda: lib.adn_render_rays_aux(h, pose, rot, d_dirs.data_ptr(), n, thr, K, d_out.data_ptr(), d_ns.data_ptr(),
                                                    None, C.byref(AuxOutputs()), None),
        "camera": lambda: lib.adn_render_camera(h, pose, rot, W, H, row0, rows, thr, K, d_out.data_ptr(), d_ns.data_ptr(), None),
        "rgba8": lambda: lib.adn_render_camera_rgba8(h, pose, rot, W, H, row0, rows, thr, K, d_out.data_ptr(), None),
        "rays_host": lambda: lib.adn_render_rays_host(h, pose, rot, h_dirs.ctypes.data, n, thr, K, h_rgb.ctypes.data, h_ns.ctypes.data),
        "camera_host": lambda: lib.adn_render_camera_host(h, pose, rot, W, H, row0, rows, thr, K, h_rgb.ctypes.data, h_ns.ctypes.data),
        "generate_ray_directions": lambda: lib.adn_generate_ray_directions(h, W, H, row0, rows, d_out.data_ptr(), None),
    }
    status = calls[entry]()
    torch.cuda.synchronize()
    return status


@pytest.mark.parametrize("entry", ["rays", "rays_aux", "camera", "rgba8", "rays_host", "camera_host", "generate_ray_directions"])
def test_render_entry_point_status_codes(entry):
    """Each render entry point rejects every invalid argument it takes with ADN_ERR_INVALID (1), a render without
    weights with ADN_ERR_NO_WEIGHTS (4), and returns ADN_OK (0) for an empty call (no rays / no rows)."""
    renders = entry != "generate_ray_directions"
    windowed = entry not in ("rays", "rays_aux", "rays_host")
    cases = [(dict(K=0), 1), (dict(thr=-0.1), 1), (dict(thr=0.0, K=8), 1)] if renders else []   # thr 0: dense, needs K 128
    if windowed:
        cases += [(dict(row0=4, rows=5), 1), (dict(rows=-1), 1)]                                # row0 + rows > H
    cases.append((dict(rows=0), 0))
    bare = _renderer(orc.SCENE_BARBERSHOP)
    assert _entry_status(bare, entry) == (4 if renders else 0)
    bare.close()
    sd0, sd1 = orc.make_weights("rand", seed=0)
    r = _renderer(orc.SCENE_BARBERSHOP, sd0, sd1)
    for args, status in cases:
        assert _entry_status(r, entry, **args) == status, args
    assert _entry_status(r, entry) == 0
    r.close()


@pytest.mark.parametrize("K", [8, 16])
def test_threshold_sweep_vs_oracle(K, pavillon_weights):
    """BASELINE config 5: thr in {0.05, 0.1, 0.2, 0.3, 0.5} with the trained Pavillon weights (ragged sample counts at
    the higher thresholds).  Compared with the CPU oracle run on this host: sample counts must agree on >= 99 % of
    the rays (a borderline logit may flip between two fp32 evaluation orders) and PSNR(ours, oracle) >= 50 dB."""
    sd0, sd1 = pavillon_weights
    scene = orc.SCENE_PAVILLON
    r = _renderer(scene, sd0, sd1)
    W = H = 800
    idx = torch.arange(0, W * H, 1237)[:512]
    dirs = torch.from_numpy(orc.generate_ray_directions(W, H, scene["fov"]).reshape(-1, 3)).float()[idx]
    pose = torch.tensor(scene["view_cell_center"]) + torch.tensor([0.05, -0.03, 0.02])
    rot = torch.tensor([[1, 0, 0], [0, 0, -1], [0, 1, 0]], dtype=torch.float32)
    for thr in (0.05, 0.1, 0.2, 0.3, 0.5):
        ref = orc.render_rays(pose, rot, dirs, sd0, sd1, scene, thr, K)
        out = r.render_rays(pose, rot, dirs.cuda(), thr, K)
        same = (out["n_samples"].cpu().long() == ref["n_samples"]).float().mean().item()
        p = orc.psnr(out["rgb"].cpu(), ref["rgb"])
        print(f"K={K} thr={thr}: mean spr {ref['n_samples'].float().mean():.2f}, identical counts {same:.4f}, PSNR {p:.2f} dB")
        assert same >= 0.99 and p >= 50.0
    r.close()


@pytest.mark.parametrize("n", [0, 1, 127, 129, 257, 385])
def test_render_ragged_sizes(n):
    """Ray counts around the 128-row tile / CTA-pair boundaries (odd tile counts leave one CTA of a pair without a
    tile) and the empty call."""
    scene = orc.SCENE_BARBERSHOP
    sd0, sd1 = orc.make_weights("shaped", seed=0)
    r = _renderer(scene, sd0, sd1)
    pose, rot = torch.tensor(scene["view_cell_center"]), torch.eye(3)
    dirs = torch.from_numpy(orc.generate_ray_directions(800, 800, scene["fov"]).reshape(-1, 3)).float()[::1663][:n]
    out = r.render_rays(pose, rot, dirs.cuda(), 0.2, 8)
    assert out["rgb"].shape == (n, 3)
    if n:
        ref = orc.render_rays(pose, rot, dirs, sd0, sd1, scene, 0.2, 8)
        assert torch.equal(out["n_samples"].cpu().long(), ref["n_samples"])
        assert np.abs(out["rgb"].cpu().numpy() - ref["rgb"].numpy()).max() < 5e-3
    r.close()


def test_image_metrics_on_device(bare):
    """adn_image_metrics == calculate_mse / calculate_psnr (src/evaluate.py:49-54)."""
    g = torch.Generator().manual_seed(11)
    a = torch.rand(800 * 800, 3, generator=g) * 1.2 - 0.1
    b = torch.rand(800 * 800, 3, generator=g)
    m = bare.image_metrics(a.cuda(), b.cuda())
    diff = (a.double() - b.double())
    mse = float(diff.pow(2).sum() / diff.numel())
    assert abs(m["mse"] - mse) < 1e-12 and abs(m["psnr"] - 10 * np.log10(1.0 / mse)) < 1e-9
    mc = bare.image_metrics(a.cuda(), b.cuda(), clamp01=True)
    d2 = a.clamp(0, 1).double() - b.double()
    assert abs(mc["mse"] - float(d2.pow(2).sum() / d2.numel())) < 1e-12
    again = bare.image_metrics(a.cuda(), b.cuda())
    assert again == m                                              # deterministic reduction
    with pytest.raises(Exception):
        bare.image_metrics(a.cuda(), b[:10].cuda())


# ------------------------------------------------------------------------------------ NDC / LLFF variant
def test_ndc_variant_stages_and_render():
    """configs/fine_training_ndc.ini: 30-feature sampling net ("2-2"), FromClassifiedDepthAdaptiveNoDepthRange (z = cell
    centre), ndc_rays + un-normalised positions in stage 3, NeRFOutputDepth = depth map -- against the reference's own
    tensors (golden case ndc_k16_t0.15)."""
    g = load_golden("ndc_k16_t0.15")
    m = g["meta"]
    K, thr, scene = m["K"], m["thr"], m["scene_params"]
    assert scene["use_ndc"] and g["x0"].shape[1] == 30
    sd0, sd1 = case_weights("ndc_k16_t0.15")
    r = _renderer(scene, sd0, sd1)
    dirs = torch.from_numpy(g["dirs"]).cuda()
    # stage 0: "2-2" encoding, direction block first
    x0, ro, rd = r.stage0(g["pose"], g["rot"], dirs)
    assert x0.shape == (g["dirs"].shape[0], 30)
    np.testing.assert_array_equal(rd.cpu().numpy(), g["ray_d"])
    np.testing.assert_allclose(ro.cpu().numpy(), g["ray_o"], rtol=0, atol=1e-6)
    np.testing.assert_allclose(x0.cpu().numpy(), g["x0"], rtol=0, atol=2e-5)
    # stage 1 on the reference's features (bf16x3 split precision, K = 30 padded)
    raw0 = r.mlp0(torch.from_numpy(g["x0"]).cuda())
    np.testing.assert_allclose(raw0.cpu().numpy(), g["raw0"], rtol=0, atol=2e-4 * max(1.0, np.abs(g["raw0"]).max()))
    # stage 2 on the reference's raw0: bit-exact selection, z = (cell + 0.5) / 128 exactly
    s2 = r.stage2(torch.from_numpy(g["raw0"]).cuda(), thr, K)
    mask, ray, z = _packed_from_golden(g, K)
    np.testing.assert_array_equal(s2["count"].cpu().numpy(), mask.sum(1))
    np.testing.assert_array_equal(s2["ray"].cpu().numpy(), ray)
    np.testing.assert_array_equal(s2["z"].cpu().numpy(), z)
    np.testing.assert_array_equal(s2["z"].cpu().numpy(), (s2["cell"].cpu().numpy() + 0.5) / 128.0)
    # stage 3: ndc_rays, no normalisation
    x1 = r.stage3(torch.from_numpy(g["ray_o"]), torch.from_numpy(g["ray_d"]), torch.from_numpy(ray.astype(np.int32)),
                  torch.from_numpy(z)).cpu().numpy()
    ref = g["x1_nan"].reshape(-1, 90)[mask.flatten()]
    err = np.abs(x1 - ref)
    assert np.abs(x1[:, :3] - ref[:, :3]).max() < 2e-5 * max(1.0, np.abs(ref[:, :3]).max())     # NDC positions
    assert err[:, 63:].max() < 2e-5                                                             # view encoding
    assert err[:, :63].max() < 5e-3, err[:, :63].max()    # 2^9 band on |x| up to ~7 (un-normalised NDC coordinates)
    # end to end + auxiliaries
    out = r.render_rays(g["pose"], g["rot"], dirs, thr, K, want_aux=True)
    ns = out["n_samples"].cpu().numpy()
    same = ns == np.round(g["asp"] * K).astype(np.int32)
    assert same.mean() >= 0.98
    rgb = out["rgb"].cpu().numpy()
    p = orc.psnr(rgb[same], g["rgb"][same])
    print(f"ndc: identical counts {same.mean():.4f}, PSNR {p:.2f} dB")
    assert p > 40.0
    np.testing.assert_allclose(out["z_vals"].cpu().numpy()[same], g["z_nan"][same], rtol=0, atol=0, equal_nan=True)
    np.testing.assert_array_equal(out["depth_est"].cpu().numpy(), out["depth_map"].cpu().numpy())   # features.py:573-574
    assert np.abs(out["depth_est"].cpu().numpy()[same] - g["depth_est"][same, 0]).max() < 5e-2
    # camera entry: the frame size feeds ndc_rays (800 x 800 here = the scene's w, h): same as explicit rays
    cam = r.render_camera(g["pose"], g["rot"], 800, 800, thr, K, row0=0, rows=4)["rgb"]
    dirs_all = torch.from_numpy(orc.generate_ray_directions(800, 800, scene["fov"]).reshape(-1, 3)).float()[:4 * 800].cuda()
    exp = r.render_rays(g["pose"], g["rot"], dirs_all, thr, K)["rgb"]
    assert torch.equal(cam, exp)
    r.close()
    # a 90-feature sampling net is rejected for this scene, with a message
    bad0, _ = orc.make_weights("rand", seed=0)
    r2 = _renderer(scene, bad0, sd1)
    with pytest.raises(Exception, match="30"):
        r2.render_rays(g["pose"], g["rot"], dirs, thr, K)
    r2.close()


def test_render_k32_uses_the_general_kernels():
    """16 < K < 128: warp-per-ray top-K (stage2_kernel) and the warp-per-ray composite, end to end against the oracle."""
    scene = orc.SCENE_BARBERSHOP
    sd0, sd1 = orc.make_weights("shaped", seed=0)
    r = _renderer(scene, sd0, sd1)
    pose, rot = torch.tensor(scene["view_cell_center"]), orc.rotation_yaw(90.0)
    dirs = torch.from_numpy(orc.generate_ray_directions(800, 800, scene["fov"]).reshape(-1, 3)).float()[::311][:2000]
    for K, thr in ((32, 0.05), (64, 0.0125), (24, 0.2)):
        ref = orc.render_rays(pose, rot, dirs, sd0, sd1, scene, thr, K)
        out = r.render_rays(pose, rot, dirs.cuda(), thr, K)
        same = (out["n_samples"].cpu().long() == ref["n_samples"]).float().mean().item()
        p = orc.psnr(out["rgb"].cpu().numpy(), ref["rgb"].numpy())
        print(f"K={K} thr={thr}: mean spr {ref['n_samples'].float().mean():.2f}, identical counts {same:.4f}, PSNR {p:.2f} dB")
        assert same >= 0.999 and p >= 49.4
    r.close()


def test_fused_input_encoder_option():
    """"fuse_encoder": stage 3 computed inside the shading kernel (same device functions, the packed bf16 input block is
    written straight to shared memory instead of the [M, 90]-sized tile buffer) -- same picture, bit for bit, adaptive and
    dense; and toggling the option leaves the default path's picture unchanged."""
    scene = orc.SCENE_BARBERSHOP
    sd0, sd1 = orc.make_weights("shaped", seed=0)
    r = _renderer(scene, sd0, sd1)
    pose, rot = torch.tensor(scene["view_cell_center"]), orc.rotation_yaw(45.0)
    new = r.render_camera(pose, rot, 800, 800, 0.2, 8, row0=100, rows=300, want_nsamples=True)
    a = r.render_camera(pose, rot, 800, 800, 0.2, 8, row0=100, rows=300, want_nsamples=True)
    d = r.render_camera(pose, rot, 800, 800, 0.0, 128, row0=0, rows=6)
    r.set_option("fuse_encoder", 1)
    b = r.render_camera(pose, rot, 800, 800, 0.2, 8, row0=100, rows=300, want_nsamples=True)
    e = r.render_camera(pose, rot, 800, 800, 0.0, 128, row0=0, rows=6)
    r.set_option("fuse_encoder", 0)
    again = r.render_camera(pose, rot, 800, 800, 0.2, 8, row0=100, rows=300, want_nsamples=True)
    assert torch.equal(a["n_samples"], b["n_samples"]) and torch.equal(a["rgb"], b["rgb"])
    assert torch.equal(d["rgb"], e["rgb"])
    assert torch.equal(a["n_samples"], new["n_samples"]) and torch.equal(a["rgb"], new["rgb"])
    assert torch.equal(again["n_samples"], new["n_samples"]) and torch.equal(again["rgb"], new["rgb"])
    r.close()
