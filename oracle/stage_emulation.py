"""fp32-FAITHFUL EMULATION OF THE SIMT STAGES -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

`oracle/adanerf_oracle.py` restates the *reference* (torch fp32), which the kernels follow only up to the last ulp of a
position (and so up to ~1e-4 on the 2^9 encoding band).  This module restates the *kernels* instead: stage 0
(`stage0_kernel`), stage 3's per-sample inputs (`sample_inputs`), the positional encoding (`posenc3`) and both stage-5
composites (`stage5_thread_kernel`, `stage5_warp_kernel`), operation for operation in numpy float32.  Every position
operation of those kernels is an explicit round-to-nearest intrinsic or an fma in a fixed order, so the emulation gives
the kernels' bits, and the GPU tests (`tests/test_stage_kernels_exact.py`) compare with `assert_array_equal`.

For stage 2 it restates the host side bit for bit: the 128-entry adaptive depth table `adn_create` uploads (`zlut`) and
the dense table of `ensure_dense_lut` (`zlut_dense`); `stage2_packed` turns the oracle's selection into the kernels'
packed buffers.

The composites return every output the kernels write (rgb, weights, alpha, z_vals, depth_map, acc_map; `stage5_dense`
for dense mode), and the per-ray epilogue is restated on its own: `disp_map` and `rgba8` exactly, `depth_est` as its exact
fp32 argument plus a float64 value with logf's bound.

What it cannot restate bit for bit is CUDA's `sincosf`, `expf` and `logf`.  So `posenc3` either takes correctly rounded float64
anchors or the kernel's own band-0 / band-5 outputs (then only the double-angle recurrence is emulated), and the
composites take the sigmoid values as an input.  The fixed-K sampler (`pdf_sample_kernel`: `pdf_sample`) and the density
composite (`density_alpha`, then the composites' `alpha=` path) take `expf` and double `pow` as callables
(tests/test_donerf_exact_gpu.py).

numpy float32 ufuncs round every operation to nearest and never contract a multiply and an add, so `a * b + c` below is
two roundings, exactly like `__fadd_rn(__fmul_rn(a, b), c)`.  Line numbers cite `adanerf_b200/csrc/`.
"""
import functools
import math

import numpy as np

F32, F64 = np.float32, np.float64
ANCHOR_EVERY = 5             # kAnchor (posenc.cuh:17)
EPS_T = F32(1e-10)           # the 1e-10f of the transmittance factor (stages.cu:983,1035)


def fma32(a, b, c):
    """Correctly rounded fp32 fma(a, b, c).  The product of two fp32 values is exact in float64 (24 + 24 <= 53 bits); the
    sum is rounded to odd in float64 (TwoSum gives the error term; an inexact sum is truncated toward zero and its last
    bit set), then rounded to fp32.  Round-to-odd at 53 >= 24 + 2 bits followed by round-to-nearest equals one rounding
    to nearest, so there is no double-rounding error."""
    a64 = np.asarray(a, F32).astype(F64)
    b64 = np.asarray(b, F32).astype(F64)
    c64 = np.asarray(c, F32).astype(F64)
    p = a64 * b64
    s = p + c64
    with np.errstate(invalid="ignore", over="ignore"):
        bp = s - p
        e = (p - (s - bp)) + (c64 - bp)
        inexact = np.isfinite(s) & (e != 0)
        away = inexact & ((e < 0) != (s < 0))          # s was rounded away from zero: truncate it
    s = np.where(away, np.nextafter(s, 0.0), s)
    s = (np.asarray(s, F64).view(np.uint64) | inexact.astype(np.uint64)).view(F64)
    return s.astype(F32)


def ulp32(y):
    """fp32 ulp at |y| (the spacing of the fp32 value nearest to y)."""
    return np.spacing(np.abs(np.asarray(y, F64)).astype(F32)).astype(F64)


# ------------------------------------------------------------------------------------------------- scene constants
def scene_constants(scene):
    """The SceneDev values adn_create derives from a scene dict (api.cu:767-780, set_ndc_projection api.cu:420-424).  The
    scene travels as fp32 fields (adn_scene), so every float is rounded to fp32 before the float64 work."""
    size = [float(F32(v)) for v in scene["view_cell_size"]]
    r2 = 0.0
    for v in size:
        r2 += (v / 2.0) * (v / 2.0)
    r = math.sqrt(r2)
    ndc = bool(scene.get("use_ndc"))
    nfp0 = scene.get("n_freq_pos0") or (2 if ndc else scene.get("n_freq_pos", 10))
    nfd0 = scene.get("n_freq_dir0") or (2 if ndc else scene.get("n_freq_dir", 4))
    out = dict(c=np.asarray(scene["view_cell_center"], F32), r2=F32(r * r),
               sqrt_max_depth=F32(math.sqrt(float(F32(scene["max_depth"])))), ndc=ndc, nfp0=int(nfp0), nfd0=int(nfd0),
               ndc_cw=F32(0), ndc_ch=F32(0))
    w, h = int(scene.get("w") or 0), int(scene.get("h") or 0)
    if ndc and w > 0 and h > 0:
        f_in = float(F32(scene.get("focal") or 0.0))
        focal = f_in if f_in > 0 else 0.5 * float(w) / math.tan(0.5 * float(F32(scene["fov"])))
        out["ndc_cw"] = F32(-1.0 / (float(w) / (2.0 * focal)))
        out["ndc_ch"] = F32(-1.0 / (float(h) / (2.0 * focal)))
    return out


# ------------------------------------------------------------------------------------------------- depth tables
def _to_world(z, scene):
    """LogTransform.to_world as adn_create / ensure_dense_lut evaluate it: pow in float64 on max_v = dr1 - dr0 (the fp32
    scene fields widened), rounded to fp32, then (w - 1) + dr0 in fp32.  NDC scenes (FromClassifiedDepthAdaptiveNoDepthRange)
    keep z itself."""
    z = np.asarray(z, F32)
    if scene.get("use_ndc"):
        return z.copy()
    dr0, dr1 = F32(scene["depth_range"][0]), F32(scene["depth_range"][1])
    base = (float(dr1) - float(dr0)) + 1.0
    w = np.array([math.pow(base, float(v)) for v in z], F64).astype(F32)
    return (w - F32(1)) + dr0


def zlut(scene):
    """The adaptive depth table (api.cu:781-789): cell centres (i + 0.5) * (1 / 128) in fp32, then _to_world.  [128] fp32."""
    return _to_world((np.arange(128, dtype=F32) + F32(0.5)) * F32(1.0 / 128.0), scene)


def linspace01(K, symmetric=True):
    """torch.linspace(0, 1, K + 1) in fp32 as ATen's CPU kernel evaluates it: k * step below the half-way index,
    fma(-step, K - k, 1) from it on, step = 1 / K -- the lin of api.cu:433-434 and linspace01 of stages.cu (the sampler's
    u and cell edges).  symmetric=False takes k * step on both halves (teeth tests).  [K + 1] fp32."""
    step = F32(1) / F32(K)
    k = np.arange(K + 1)
    if not symmetric:
        return (k.astype(F32) * step).astype(F32)
    return np.where(k < (K + 1) // 2, k.astype(F32) * step, fma32(-step, (K - k).astype(F32), F32(1))).astype(F32)


def zlut_dense(scene, K):
    """The dense table of ensure_dense_lut (api.cu:426-439): t = linspace01(K)[:K] + fp32(0.5 / K), z = z_near (1 - t) +
    z_far t in fp32, then _to_world.  [K] fp32."""
    t = linspace01(K)[:K] + F32(0.5 / K)
    near, far = F32(scene.get("z_near", 0.001)), F32(scene.get("z_far", 1.0))
    return _to_world(near * (F32(1) - t) + far * t, scene)


# ------------------------------------------------------------------------------------------------------- stage 2
def stage2_packed(sel, lut):
    """The packed buffers of stage 2 (stage2_kernel / stage2_thread_kernel, stages.cu) from the selection of
    orc.stage2_sample (`sel`: count [N], cell [N,K] ascending, -1 padded, zp [N,K]): ray-major, cells ascending inside a ray.
    -> dict(count [N], offset [N], total, ray [M], cell [M], zp [M], z [M] = lut[cell]); int32 / fp32 like the kernels'."""
    cell = np.asarray(sel["cell"])
    live = cell >= 0
    count = live.sum(1).astype(np.int32)
    assert np.array_equal(count, np.asarray(sel["count"])), "stage2_packed: counts disagree with the selection"
    offset = (np.cumsum(count, dtype=np.int64) - count).astype(np.int32)
    c = cell[live].astype(np.int32)
    return dict(count=count, offset=offset, total=int(count.sum()),
                ray=np.repeat(np.arange(cell.shape[0], dtype=np.int32), count), cell=c,
                zp=np.asarray(sel["zp"], F32)[live], z=np.asarray(lut, F32)[c])


# ------------------------------------------------------------------------------------------------------- stage 0a
def pixel_dir(W, H, fov, row0=0, rows=None):
    """gen_dirs_kernel / pixel_dir (stages.cu:22-32) with camera_rays' float64 constants (api.cu:455-472): [rows*W, 3]."""
    rows = H - row0 if rows is None else rows
    fov = float(F32(fov))
    focal = 0.5 * W / math.tan(0.5 * fov)
    x_dist = math.tan(fov / 2) * focal
    y_dist = x_dist * (float(H) / float(W))
    x_pp, y_pp = x_dist / (W / 2.0), y_dist / (H / 2.0)
    start_x, start_y = -(x_dist - x_pp / 2), -(y_dist - y_pp / 2)
    rx = np.broadcast_to(start_x + x_pp * np.arange(W, dtype=F64), (rows, W))
    ry = np.broadcast_to((start_y + y_pp * np.arange(row0, row0 + rows, dtype=F64))[:, None], (rows, W))
    n = np.sqrt((rx * rx + ry * ry) + focal * focal)
    d = np.stack([(rx / n).astype(F32), -(ry / n).astype(F32), -(focal / n).astype(F32)], -1)
    return d.reshape(-1, 3)


# ---------------------------------------------------------------------------------------------------- posenc3
def posenc3(v, L, anchors=None, anchor_every=ANCHOR_EVERY):
    """posenc3<L> (posenc.cuh:18-40): [..., 3] -> [..., 3 + 6L] = [v, sin 2^0 v, cos 2^0 v, ..., sin 2^(L-1) v, ...].
    Bands f % 5 == 0 are anchors: with anchors=None the correctly rounded float64 sin / cos of the exact fp32 argument
    v * 2^f; otherwise the columns of `anchors` (the kernel's own [..., 3 + 6L] block), so that only the recurrence is
    emulated.  Every other band is the double-angle step from the band below: s' = (2s) c (2s is exact), c' = fma(-2s, s, 1).
    anchor_every: the anchor spacing (a larger value removes the band-5 anchor; only the teeth tests change it)."""
    v = np.asarray(v, F32)
    out = np.empty(v.shape[:-1] + (3 + 6 * L,), F32)
    out[..., :3] = v
    s = c = None
    for f in range(L):
        lo = 3 + 6 * f
        if f % anchor_every == 0:
            if anchors is None:
                x = (v * F32(2.0 ** f)).astype(F64)
                s, c = np.sin(x).astype(F32), np.cos(x).astype(F32)
            else:
                s, c = np.asarray(anchors[..., lo:lo + 3], F32), np.asarray(anchors[..., lo + 3:lo + 6], F32)
        else:
            s, c = (F32(2) * s) * c, fma32(F32(-2) * s, s, F32(1))
        out[..., lo:lo + 3] = s
        out[..., lo + 3:lo + 6] = c
    return out


def posenc_f64(v, L):
    """The encoding evaluated in float64 on the exact fp32 inputs (the reference every band's error is measured against)."""
    v = np.asarray(v, F32).astype(F64)
    out = np.empty(v.shape[:-1] + (3 + 6 * L,), F64)
    out[..., :3] = v
    for f in range(L):
        out[..., 3 + 6 * f:6 + 6 * f] = np.sin(v * 2.0 ** f)
        out[..., 6 + 6 * f:9 + 6 * f] = np.cos(v * 2.0 ** f)
    return out


@functools.lru_cache(maxsize=None)
def recurrence_band_bounds(L=10, n_args=1 << 17, max_ulps=2, seed=0):
    """Per band f: the largest |posenc3 - float64| over n_args fp32 arguments in [-4, 4] (more than a turn of every
    anchor angle) when each anchor value, sin and cos independently, is any fp32 value within max_ulps ulp of the
    correctly rounded one -- everything posenc3 can return while sincosf keeps its documented 2-ulp bound (CUDA C++
    Programming Guide, single-precision mathematical functions).  Bands f and f +- 5 see the same recurrence, so each
    takes the larger of the two.  Returns a float64 array [L]."""
    rng = np.random.default_rng(seed)
    x = rng.uniform(-4.0, 4.0, n_args).astype(F32)
    steps = range(-max_ulps, max_ulps + 1)
    worst = np.zeros(L, F64)
    for f0 in range(0, L, ANCHOR_EVERY):
        arg = x * F32(2.0 ** f0)
        a64 = arg.astype(F64)
        s0, c0 = np.sin(a64).astype(F32), np.cos(a64).astype(F32)
        s_opts = [_nudge(s0, k) for k in steps]
        c_opts = [_nudge(c0, k) for k in steps]
        s = np.concatenate([so for so in s_opts for _ in c_opts])
        c = np.concatenate([co for _ in s_opts for co in c_opts])
        ref = np.tile(a64, len(s_opts) * len(c_opts))
        for f in range(f0, min(L, f0 + ANCHOR_EVERY)):
            if f > f0:
                s, c = (F32(2) * s) * c, fma32(F32(-2) * s, s, F32(1))
            r = ref * 2.0 ** (f - f0)
            worst[f] = max(np.abs(s - np.sin(r)).max(), np.abs(c - np.cos(r)).max())
    for f in range(L):
        for g in (f - ANCHOR_EVERY, f + ANCHOR_EVERY):
            if 0 <= g < L:
                worst[f] = max(worst[f], worst[g])
    return worst


def _nudge(x, k):
    """x moved by k fp32 ulps."""
    x = np.asarray(x, F32)
    for _ in range(abs(k)):
        x = np.nextafter(x, F32(np.inf) if k > 0 else F32(-np.inf))
    return x


# ------------------------------------------------------------------------------------------------------- stage 0b
def _dot3(a, b):
    """((a0 b0 + a1 b1) + a2 b2), every operation rounded (stages.cu:80-81,87)."""
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def rotate(rot, dirs):
    """nds = R d as the FMA chain fma(R[r,2], d2, fma(R[r,1], d1, R[r,0] d0)) (stages.cu:73-75)."""
    R = np.asarray(rot, F32).reshape(9)
    d = np.asarray(dirs, F32).reshape(-1, 3)
    return np.stack([fma32(R[3 * r + 2], d[:, 2], fma32(R[3 * r + 1], d[:, 1], R[3 * r] * d[:, 0])) for r in range(3)], -1)


def sphere_delta(pose, nds, scene):
    """compute_ray_offset's discriminant delta = udot^2 - (|o - c|^2 - r^2) (stages.cu:79-82); <= 0 is clamped to 0."""
    k = scene_constants(scene)
    omc = np.asarray(pose, F32).reshape(3) - k["c"]
    udot = _dot3(omc[None, :], nds)
    return udot, udot * udot - (_dot3(omc, omc) - k["r2"])


def stage0(pose, rot, dirs, scene, nfd=None, nfp=None, contract=False):
    """stage0_kernel<false, NFD, NFP> (stages.cu:52-111) -> (ray_o [N,3], ray_d [N,3], x0 [N, 6 + 6 (NFD + NFP)]) with the
    direction block first.  nfd / nfp default to the scene's sampling-net encoding ("10-4", or "2-2" with NDC).
    contract=True evaluates p = pose + nds t as one fma (a kernel the compiler was allowed to contract; teeth tests)."""
    k = scene_constants(scene)
    nfd = k["nfd0"] if nfd is None else nfd
    nfp = k["nfp0"] if nfp is None else nfp
    pose = np.asarray(pose, F32).reshape(3)
    nds = rotate(rot, dirs)
    udot, delta = sphere_delta(pose, nds, scene)
    t = -udot + np.sqrt(np.fmax(delta, F32(0)))                                  # :83
    if contract:
        p = np.stack([fma32(nds[:, a], t, pose[a]) for a in range(3)], -1)
    else:
        p = pose[None, :] + nds * t[:, None]                                    # :86
    nn = np.sqrt(_dot3(nds, nds))                                               # :87
    dn = nds / nn[:, None]                                                      # :90
    x0 = np.concatenate([posenc3(dn, nfd), posenc3(p, nfp)], -1)                 # :91-92
    return p, nds, x0


# -------------------------------------------------------------------------------------------------------- stage 3
def sample_inputs(scene, ray_o, ray_d, ray_idx, z, contract=False):
    """sample_inputs (posenc.cuh:45-84) for samples (ray_idx, z) -> (pos [M,3], dir [M,3]): the NDC branch (ndc_rays with
    near = 1, un-normalised position, direction d' / |d'|) or pos - c over sqrt(max_depth) sqrt|pos - c| with the raw
    direction.  contract=True fuses o + d z into one fma (teeth tests)."""
    k = scene_constants(scene)
    r = np.asarray(ray_idx, np.int64)
    o = np.asarray(ray_o, F32).reshape(-1, 3)[r]
    d = np.asarray(ray_d, F32).reshape(-1, 3)[r]
    zw = np.asarray(z, F32)
    if k["ndc"]:
        cw, ch = k["ndc_cw"], k["ndc_ch"]
        t = -(F32(1) + o[:, 2]) / d[:, 2]                                        # :57
        on = o + t[:, None] * d                                                  # :60
        q0, q1 = on[:, 0] / on[:, 2], on[:, 1] / on[:, 2]
        o0, o1 = (cw * on[:, 0]) / on[:, 2], (ch * on[:, 1]) / on[:, 2]
        o2 = F32(1) + F32(2) / on[:, 2]
        d0 = cw * (d[:, 0] / d[:, 2] - q0)
        d1 = ch * (d[:, 1] / d[:, 2] - q1)
        d2 = F32(-2) / on[:, 2]
        oo, dd = np.stack([o0, o1, o2], -1), np.stack([d0, d1, d2], -1)
        pos = fma32(dd, zw[:, None], oo) if contract else oo + dd * zw[:, None]  # :68-70
        dn = np.sqrt(_dot3(dd, dd))                                              # :71
        return pos, dd / dn[:, None]                                             # :72-74
    pos = (fma32(d, zw[:, None], o) if contract else o + d * zw[:, None]) - k["c"][None, :]   # :77
    nrm = np.sqrt(_dot3(pos, pos))                                               # :79
    den = k["sqrt_max_depth"] * np.sqrt(nrm)                                     # :80
    with np.errstate(invalid="ignore", divide="ignore"):
        return pos / den[:, None], d                                             # :82


def stage3(scene, ray_o, ray_d, ray_idx, z):
    """stage3_kernel's x1 [M, 90] (stages.cu:869-898) with float64 anchors: the position block (10 bands) first."""
    pos, d = sample_inputs(scene, ray_o, ray_d, ray_idx, z)
    with np.errstate(invalid="ignore"):
        return np.concatenate([posenc3(pos, 10), posenc3(d, 4)], -1)


# -------------------------------------------------------------------------------------------------------- stage 5
NAN32 = np.uint32(0x7fc00000).view(F32)    # the NaN the kernels write (and torch's float("nan"))


def _gather(a, idx, live, fill=0):
    a = np.asarray(a)
    if a.shape[0] == 0:
        return np.full(idx.shape + a.shape[1:], fill, a.dtype)
    return a[np.where(live, idx, 0)]


def _z_vals(z, live, dense=False):
    """The z_vals slots (s5_z_val): NaN where not live and -- the reference's adaptive path (features.py:546-547) -- where
    z == +-0; dense mode keeps z."""
    return np.where(live & (dense | (z != 0)), z, NAN32).astype(F32)


def stage5_thread(sig, zp, z, offset, count, K, eps=EPS_T, alpha=None):
    """stage5_thread_kernel (stages.cu) on sigmoid values sig [M,4] (rgb, alpha): per ray the sequential chain
    alpha = s_a zp, w = alpha T, T = T ((1 - alpha) + 1e-10), c += w s, depth += w z, acc += w.  -> dict(rgb [N,3],
    weights / alpha [N,K] zero padded, z_vals [N,K] NaN padded, depth_map [N], acc_map [N]).  eps: the 1e-10 term (teeth
    tests drop it).  alpha: per-sample alpha [M] (the density composite, stage5_thread_kernel<true>: see density_alpha);
    then sig's fourth column and zp are not read and z_vals keeps z == 0."""
    sig, z = np.asarray(sig, F32), np.asarray(z, F32)
    given = alpha is not None
    zp = np.asarray(alpha if given else zp, F32)
    off, cnt = np.asarray(offset, np.int64), np.asarray(count, np.int64)
    n = cnt.shape[0]
    T = np.ones(n, F32)
    acc = np.zeros((n, 5), F32)          # r, g, b, depth, acc
    w_out = np.zeros((n, K), F32)
    a_out = np.zeros((n, K), F32)
    z_out = np.full((n, K), NAN32, F32)
    with np.errstate(invalid="ignore", over="ignore"):
        for j in range(K):
            live = j < cnt
            if not live.any():
                break
            idx = off + j
            s = _gather(sig, idx, live)
            zz = _gather(z, idx, live)
            a = _gather(zp, idx, live) if given else s[:, 3] * _gather(zp, idx, live)
            w = a * T
            T = np.where(live, T * ((F32(1) - a) + eps), T)
            terms = np.concatenate([w[:, None] * s[:, :3], (w * zz)[:, None], w[:, None]], -1)
            acc = np.where(live[:, None], acc + terms, acc)
            w_out[:, j] = np.where(live, w, F32(0))
            a_out[:, j] = np.where(live, a, F32(0))
            z_out[:, j] = _z_vals(zz, live, given)
    return dict(rgb=acc[:, :3].copy(), weights=w_out, alpha=a_out, z_vals=z_out, depth_map=acc[:, 3].copy(),
                acc_map=acc[:, 4].copy())


def stage5_warp(sig, zp, z, offset, count, K, eps=EPS_T, tree=True, dense=False, alpha=None, butterfly=True):
    """stage5_warp_kernel (stages.cu), as lane 0 ends it: per 32-sample block a Hillis-Steele inclusive product scan of
    f = (1 - alpha) + 1e-10 (lane l multiplies in lane l - o's value, o = 1, 2, 4, 8, 16), T = carry * (exclusive
    product), w = alpha T, carry *= the block's product; each lane sums its own w s / w z / w over the blocks, then an xor
    butterfly (o = 16 ... 1) adds the lanes.  Lanes past the ray's count take alpha = s = z = 0.  Same outputs as
    stage5_thread.  tree=False takes T as the sequential product instead, butterfly=False adds the lanes' sums in lane
    order (teeth tests).  dense: z_vals keeps z == 0 (stage5_dense passes the dense layout).  alpha: per-sample alpha [M]
    (the density composite, stage5_warp_kernel<true>), as in stage5_thread."""
    sig, z = np.asarray(sig, F32), np.asarray(z, F32)
    given = alpha is not None
    zp = np.asarray(alpha if given else zp, F32)
    dense = dense or given
    off, cnt = np.asarray(offset, np.int64), np.asarray(count, np.int64)
    n = cnt.shape[0]
    lanes = np.arange(32)
    carry = np.ones(n, F32)
    acc = np.zeros((n, 32, 5), F32)      # per lane: r, g, b, depth, acc
    w_out = np.zeros((n, K), F32)
    a_out = np.zeros((n, K), F32)
    z_out = np.full((n, K), NAN32, F32)
    with np.errstate(invalid="ignore", over="ignore"):
        for j0 in range(0, int(cnt.max(initial=0)), 32):
            run = j0 < cnt                                               # rays whose loop reaches this block
            j = j0 + lanes[None, :]
            live = j < cnt[:, None]
            idx = off[:, None] + j
            s = np.where(live[..., None], _gather(sig, idx, live), F32(0))
            alpha = np.where(live, _gather(zp, idx, live) if given else s[..., 3] * _gather(zp, idx, live), F32(0))
            zz = np.where(live, _gather(z, idx, live), F32(0))
            f = (F32(1) - alpha) + eps
            if tree:
                p = f.copy()
                for o in (1, 2, 4, 8, 16):
                    p[:, o:] = p[:, o:] * p[:, :-o]
            else:
                p = np.empty_like(f)
                p[:, 0] = f[:, 0]
                for l in range(1, 32):
                    p[:, l] = p[:, l - 1] * f[:, l]
            excl = np.concatenate([np.ones((n, 1), F32), p[:, :31]], 1)
            T = carry[:, None] * excl
            w = alpha * T
            terms = np.stack([w * s[..., 0], w * s[..., 1], w * s[..., 2], w * zz, w], -1)
            acc = np.where(run[:, None, None], acc + terms, acc)
            carry = np.where(run, carry * p[:, 31], carry)
            inside = j0 + lanes < K
            cols = j0 + lanes[inside]
            w_out[:, cols] = np.where(live & run[:, None], w, F32(0))[:, inside]
            a_out[:, cols] = np.where(live & run[:, None], alpha, F32(0))[:, inside]
            z_out[:, cols] = _z_vals(zz, live & run[:, None], dense)[:, inside]
        if butterfly:
            for o in (16, 8, 4, 2, 1):
                acc = acc + acc[:, lanes ^ o]
        else:
            for l in range(1, 32):
                acc[:, 0] = acc[:, 0] + acc[:, l]
    return dict(rgb=acc[:, 0, :3].copy(), weights=w_out, alpha=a_out, z_vals=z_out, depth_map=acc[:, 0, 3].copy(),
                acc_map=acc[:, 0, 4].copy())


def stage5_dense(sig, raw0, lut):
    """stage5_warp_kernel with dense = 1: ray r's K = 128 samples are rows r * 128 + k of sig, zp = raw0 [N,128] and
    z = lut[k] (zlut_dense(scene, 128)); no padding, and z_vals keeps z == 0 (RayMarchFromPoses without remapping stores
    the z it sampled, features.py:487-491)."""
    raw0 = np.asarray(raw0, F32)
    n, K = raw0.shape
    z = np.tile(np.asarray(lut, F32), n)
    return stage5_warp(sig, raw0.reshape(-1), z, np.arange(n, dtype=np.int64) * K, np.full(n, K, np.int64), K, dense=True)


def stage5(sig, zp, z, offset, count, K):
    """The composite launch_stage5 picks for a packed (non-dense) call: the warp kernel when K > 32."""
    return (stage5_warp if K > 32 else stage5_thread)(sig, zp, z, offset, count, K)


# ------------------------------------------------------------------------------------------- stage 5 per-ray epilogue
def disp_map(dm, acc):
    """s5_write_ray_aux's disparity, the reference's 1 / torch.max(1e-10, dm / acc) (nerf_raymarch_common.py:138):
    torch.max propagates a NaN quotient (0 / 0 at acc == 0) where fmaxf would return 1e-10."""
    dm, acc = np.asarray(dm, F32), np.asarray(acc, F32)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        q = dm / acc
        return (F32(1) / np.where(np.isnan(q), q, np.fmax(F32(1e-10), q))).astype(F32)


def log_range(scene):
    """Stage5Aux.log_range (stage5_aux, api.cu): float(log(double(dr1) - double(dr0) + 1)) of the fp32 scene fields."""
    dr0, dr1 = F32(scene["depth_range"][0]), F32(scene["depth_range"][1])
    return F32(math.log(float(dr1) - float(dr0) + 1.0))


def depth_est_arg(dm, scene):
    """The exact part of the log-warped depth (LogTransform.from_world): x = max-clamped (dm - dr0) + 1 in fp32, the
    d <= 0 -> 0.001 rule included.  depth_est = logf(x) / log_range."""
    dm = np.asarray(dm, F32)
    with np.errstate(invalid="ignore", over="ignore"):
        d = dm - F32(scene["depth_range"][0])
        d = np.where(d <= 0, F32(0.001), d).astype(F32)
        return (d + F32(1)).astype(F32)


def depth_est_f64(dm, scene):
    """(value, bound): log(x) / log_range in float64 on the exact fp32 x of depth_est_arg, and the kernel's largest
    distance from it -- logf within 1 ulp (CUDA C++ Programming Guide, single-precision mathematical functions) scaled
    by 1 / log_range, plus the final __fdiv_rn's rounding (half an ulp; a whole one is allowed so that a quotient on a
    power of two may round to either side of it).  With NDC the kernel writes depth_map itself (bound 0)."""
    dm = np.asarray(dm, F32)
    if scene.get("use_ndc"):
        return dm.astype(F64), np.zeros(dm.shape, F64)
    L = float(log_range(scene))
    with np.errstate(invalid="ignore", divide="ignore"):
        y = np.log(depth_est_arg(dm, scene).astype(F64))
        v = y / L
        return v, ulp32(y) / L + ulp32(v)


def rgba8(rgb):
    """to_rgba8 / the viewer's pixel (adaptive_cuda_kernels.cu:846-851): per channel trunc(saturate(x) * 255), alpha 255.
    saturate is __saturatef -- x clamped to [+0, 1], NaN -> +0 -- the single FADD.SAT nvcc makes of helper_math.h's
    clamp fmaxf(0, fminf(x, 1)) (whose C semantics would give NaN -> 1).  [N,3] fp32 -> [N,4] uint8."""
    x = np.asarray(rgb, F32).reshape(-1, 3)
    v = np.where(x > 0, np.fmin(x, F32(1)), F32(0)) * F32(255)
    out = np.full((x.shape[0], 4), 255, np.uint8)
    out[:, :3] = np.trunc(v).astype(np.uint8)
    return out


# ------------------------------------------------------------------------------------------------- fixed-K sampler
# pdf_sample_kernel and the density composite (option "sampler" = 1).  CUDA's expf and double pow cannot be restated in
# numpy, so they are callables: expf(x) takes an fp32 array and returns fp32, pow64(base, x) takes a Python float and an
# fp32 array and returns the powers (rounded to fp32 here).  The CPU tests pass float64-rounded ones, the GPU tests
# torch's own CUDA kernels, after checking that those give the kernels' bits.
LANES = np.arange(32)


def _lane_sum64(v):
    """warp_sum_f64 of stages.cu over [N, 128]: each lane adds its four cells to 0.0 in double in order, then an xor
    butterfly (o = 16 ... 1) adds the lanes (every lane ends with the same value).  -> [N] float64."""
    v = np.asarray(v).reshape(-1, 32, 4).astype(F64)
    s = ((((F64(0) + v[..., 0]) + v[..., 1]) + v[..., 2]) + v[..., 3])
    for o in (16, 8, 4, 2, 1):
        s = s + s[:, LANES ^ o]
    return s[:, 0]


def pdf_transform(raw0, transform, expf):
    """The transform of pdf_sample_kernel: 1 = sigmoid 1 / (1 + expf(-x)) (sigmoidf_acc), 2 = softmax: the fmaxf warp
    max (NaN-ignoring, unlike torch.max), expf(x - m), the double sum (_lane_sum64), inv = 1 / float(sum), then w inv.
    raw0 [N,128] -> [N,128] fp32."""
    x = np.asarray(raw0, F32).reshape(-1, 128)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        if transform == 1:
            return F32(1) / (F32(1) + np.asarray(expf(-x), F32))
        if transform != 2:
            raise ValueError("transform must be 1 (sigmoid) or 2 (softmax)")
        m = np.fmax.reduce(x, axis=1) if x.shape[0] else np.zeros(0, F32)
        e = np.asarray(expf(x - m[:, None]), F32)
        inv = F32(1) / _lane_sum64(e).astype(F32)
        return e * inv[:, None]


def pdf_cdf(w, wsum="warp", scan="warp"):
    """The CDF pdf_sample_kernel stages in shared memory, from the transformed weights w [N,128]: w + 1e-5f, wsum =
    float(_lane_sum64(w)), pdf = w / wsum in fp32, then each lane's running double sum of its four pdf entries, a
    Hillis-Steele inclusive scan of the lanes' totals (o = 1 ... 16), and cdf[4l + k + 1] = float(excl + a[k]); cdf[0] = 0.
    -> [N,129] fp32.
    wsum: "warp", "fp32" (a sequential fp32 sum: teeth) or a callable w -> [N] (the reference's own sum).  scan: "warp",
    "fp32" (the same association in fp32: teeth) or "seq" (one sequential double cumsum, ATen's CPU cumsum)."""
    w = np.asarray(w, F32).reshape(-1, 128) + F32(1e-5)
    n = w.shape[0]
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        if callable(wsum):
            ws = np.asarray(wsum(w), F32)
        elif wsum == "fp32":
            ws = np.zeros(n, F32)
            for k in range(128):
                ws = ws + w[:, k]
        else:
            ws = _lane_sum64(w).astype(F32)
        pdf = w / ws[:, None]
        cdf = np.zeros((n, 129), F32)
        if scan == "seq":
            cdf[:, 1:] = np.cumsum(pdf.astype(F64), axis=1).astype(F32)
            return cdf
        T = F32 if scan == "fp32" else F64
        p = pdf.reshape(n, 32, 4).astype(T)
        a = np.empty_like(p)
        run = np.zeros((n, 32), T)
        for k in range(4):
            run = run + p[..., k]
            a[..., k] = run
        inc = run.copy()
        for o in (1, 2, 4, 8, 16):
            inc[:, o:] = inc[:, o:] + inc[:, :-o]
        excl = np.concatenate([np.zeros((n, 1), T), inc[:, :31]], 1)
        cdf[:, 1:] = (excl[..., None] + a).reshape(n, 128).astype(F32)
    return cdf


def _search(cdf, u, right=True):
    """The kernel's binary search over the staged cdf: the first index in [0, 129) whose entry is > u (right=True) or
    >= u (right=False), 129 if none.  Rows whose cdf is non-decreasing and NaN-free take the exact counting shortcut
    (that index is the number of entries <= u, resp. < u: one np.searchsorted of every entry into u); the others -- NaN
    or a decreasing step, where the search's path decides -- run the search itself.  cdf [N,129], u [K] ascending -> [N,K]."""
    n, K = cdf.shape[0], u.shape[0]
    lo = np.zeros((n, K), np.int64)
    with np.errstate(invalid="ignore"):
        mono = ~np.isnan(cdf).any(1) & (np.diff(cdf, axis=1) >= 0).all(1)
    m = np.nonzero(mono)[0]
    if m.size:
        k = np.searchsorted(u, cdf[m], side="left" if right else "right")     # entry i is <= u_j (< u_j) for j >= k_i
        hist = np.bincount((np.arange(m.size)[:, None] * (K + 1) + k).ravel(), minlength=m.size * (K + 1))
        lo[m] = np.cumsum(hist.reshape(m.size, K + 1), axis=1)[:, :K]
    o = np.nonzero(~mono)[0]
    if o.size:
        lo[o] = binary_search(cdf[o], u, right)
    return lo


def binary_search(cdf, u, right=True):
    """The kernel's search itself, step for step (lo = 0, hi = 129; mid = (lo + hi) >> 1; hi = mid where cdf[mid] > u,
    else lo = mid + 1), on every row.  cdf [N,129], u [K] -> [N,K]."""
    n, K = cdf.shape[0], u.shape[0]
    a = np.zeros((n, K), np.int64)
    b = np.full((n, K), 129, np.int64)
    rows = np.arange(n)[:, None]
    while (a < b).any():
        act = a < b
        mid = np.minimum((a + b) >> 1, 128)
        with np.errstate(invalid="ignore"):
            p = cdf[rows, mid] > u if right else cdf[rows, mid] >= u
        b = np.where(act & p, mid, b)
        a = np.where(act & ~p, mid + 1, a)
    return a


def depth_base(scene):
    """wbase of launch_pdf_sample (depth_base, api.cu:602): double(dr1) - double(dr0) + 1 of the fp32 scene fields."""
    dr0, dr1 = F32(scene["depth_range"][0]), F32(scene["depth_range"][1])
    return float(dr1) - float(dr0) + 1.0


def pdf_place(cdf, K, scene, pow64, right=True, clamp=True, symmetric=True):
    """Sample placement of pdf_sample_kernel for samples j = 1 .. K: u = linspace01(K + 1)[j], the search, below =
    max(0, lo - 1), above = min(128, lo), the cell edges linspace01(128), denom = c1 - c0 (1 where < 1e-5), t = (u - c0) /
    denom, zs = b0 + t (b1 - b0), then to_world: float(pow64(wbase, zs)) - 1 + dr0 in fp32.  cdf [N,129] -> z [N,K].
    right=False, clamp=False and symmetric=False are the teeth tests' mutations."""
    cdf = np.asarray(cdf, F32)
    u = linspace01(K + 1, symmetric)[1:K + 1]
    edges = linspace01(128, symmetric)
    lo = _search(cdf, u, right)
    below, above = np.maximum(lo - 1, 0), np.minimum(lo, 128)
    rows = np.arange(cdf.shape[0])[:, None]
    c0, c1 = cdf[rows, below], cdf[rows, above]
    b0, b1 = edges[below], edges[above]
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        denom = c1 - c0
        if clamp:
            denom = np.where(denom < F32(1e-5), F32(1), denom).astype(F32)
        t = (u - c0) / denom
        zs = b0 + t * (b1 - b0)
        w = np.asarray(pow64(depth_base(scene), zs)).astype(F32)
        return (w - F32(1)) + F32(scene["depth_range"][0])


def pdf_sample(raw0, K, transform, scene, expf, pow64, **teeth):
    """pdf_sample_kernel: raw0 [N,128] -> world z [N,K] (pdf_transform, pdf_cdf, pdf_place).  teeth: wsum / scan of
    pdf_cdf, right / clamp / symmetric of pdf_place."""
    cdf = pdf_cdf(pdf_transform(raw0, transform, expf), **{k: teeth.pop(k) for k in ("wsum", "scan") if k in teeth})
    return pdf_place(cdf, K, scene, pow64, **teeth)


def density_alpha(raw1_a, z, ray_d, K, expf):
    """nerf_alpha of stages.cu per sample: norm = sqrt((x^2 + y^2) + z^2) of ray_d in fp32, dist = (z[k+1] - z[k]) norm
    (1e10 norm for the last sample), relu keeping NaN, alpha = 1 - expf(-relu(a) dist); 0 at K = 1.  raw1_a [N K], z
    [N K], ray_d [N,3] -> alpha [N K] fp32 (the alpha= of stage5_thread / stage5_warp)."""
    a = np.asarray(raw1_a, F32).reshape(-1, K)
    zz = np.asarray(z, F32).reshape(-1, K)
    d = np.asarray(ray_d, F32).reshape(-1, 3)
    if K == 1:
        return np.zeros(a.size, F32)
    with np.errstate(invalid="ignore", over="ignore"):
        norm = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
        dist = np.concatenate([zz[:, 1:] - zz[:, :-1], np.full((zz.shape[0], 1), 1e10, F32)], 1) * norm[:, None]
        ra = np.where(np.isnan(a), a, np.fmax(a, F32(0)))
        return (F32(1) - np.asarray(expf(-ra * dist), F32)).reshape(-1)


def stage5_density(sig, alpha, z, K):
    """The density composite launch_stage5 picks (stage5_warp_kernel<true> when K > 32) over N rays of K samples at
    offset r K: sig [N K, 3+] the rgb sigmoids, alpha from density_alpha."""
    n = np.asarray(z).size // K
    fn = stage5_warp if K > 32 else stage5_thread
    return fn(sig, None, z, np.arange(n, dtype=np.int64) * K, np.full(n, K, np.int64), K, alpha=alpha)
