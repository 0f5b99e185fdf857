"""Selection bit for bit at frame scale: stage 2 (which cells each ray samples, how many, where they land in the packed
buffers, and their depth), the depth tables it and dense mode read, and the sample-budget select.

Everything is compared with a plain CPU restatement:
  * stage 2 with oracle.stage2_sample (stable descending sort, ties to the lower cell) turned into the kernels' packed
    buffers by stage_emulation.stage2_packed, and z with the host's depth tables stage_emulation.zlut / zlut_dense;
  * the budget threshold with budget_threshold (tests/test_sample_budget_oracle.py), and through stage 2 itself: M(t*) <= B
    and M(t* - 1 ulp) > B.
All comparisons are bit for bit."""
import numpy as np
import pytest
import torch

from conftest import load_pavillon_weights
from oracle import adanerf_oracle as orc
from oracle import stage_emulation as se
from test_sample_budget_oracle import budget_threshold

pytestmark = pytest.mark.gpu

F32 = np.float32
W = H = 800
KS = [1, 2, 8, 9, 16, 17, 32, 100, 127, 128]
SCENES = {"barbershop": orc.SCENE_BARBERSHOP, "pavillon": orc.SCENE_PAVILLON, "pavillon_ndc": orc.SCENE_PAVILLON_NDC}


def _renderer(scene, sd0=None, sd1=None):
    from adanerf_b200 import Renderer
    return Renderer(scene, device=0, sampling_net=sd0, shading_net=sd1)


def _bits(a):
    return np.ascontiguousarray(np.asarray(a, F32)).view(np.uint32)


def _weights(name):
    if name.startswith("pavillon_ndc"):
        return orc.make_weights("ndc", seed=0)
    if name.startswith("pavillon"):
        return load_pavillon_weights()
    return orc.make_weights("shaped", seed=0)


def check_stage2(r, raw0_dev, raw0, thr, K, lut, what):
    """r.stage2 against the emulation, every packed buffer bit for bit.  Returns the device result."""
    s2 = r.stage2(raw0_dev, thr, K)
    want = se.stage2_packed(orc.stage2_sample(raw0, thr, K, None, no_depth_range=True), lut)
    assert s2["total"] == want["total"], what
    for k in ("count", "offset", "ray", "cell"):
        np.testing.assert_array_equal(s2[k].cpu().numpy(), want[k], err_msg=f"{what}: {k}")
    for k in ("zp", "z"):
        np.testing.assert_array_equal(_bits(s2[k].cpu().numpy()), _bits(want[k]), err_msg=f"{what}: {k}")
    return s2


# ---------------------------------------------------------------------------------------- stage 2 on whole frames
# (scene, weights, pose offset from the view-cell centre, yaw in degrees)
FRAMES = {"pav_a": ("pavillon", (0.05, -0.03, 0.02), 0.0), "pav_b": ("pavillon", (-0.2, 0.15, -0.05), 140.0),
          "shaped": ("barbershop", (0.3, -0.2, 0.1), 35.0), "rand": ("barbershop", (0.0, 0.0, 0.0), 0.0),
          "ndc": ("pavillon_ndc", (0.02, 0.02, 0.0), 10.0)}


def _frame_raw0(name):
    scene_name, off, yaw = FRAMES[name]
    scene = SCENES[scene_name]
    sd0 = orc.make_weights("rand", seed=0)[0] if name == "rand" else _weights(scene_name)[0]
    r = _renderer(scene, sd0)
    pose = np.asarray(scene["view_cell_center"], F32) + np.asarray(off, F32)
    x0, _, _ = r.stage0(pose, orc.rotation_yaw(yaw), r.generate_ray_directions(W, H))
    raw0 = r.mlp0(x0).cpu()
    r.close()
    return raw0


def _with_extreme_rows(raw0):
    """Rows r = 5 and 21 (mod 32) moved wholly above / below every threshold (a constant per row, so their ranking and
    ties stay the net's): at large K a real sampling net has no ray with more than K cells >= a positive threshold and none
    with no cell above one at the same time, and every case should hold rays of all three kinds."""
    v = raw0.clone()
    top = float(v.max()) + 1.0
    r = torch.arange(v.shape[0])
    up, down = r % 32 == 5, r % 32 == 21
    v[up] = (v[up] - v[up].min(1, keepdim=True).values) + top
    v[down] = (v[down] - v[down].max(1, keepdim=True).values) - 1.0
    return v


@pytest.fixture(scope="module")
def frames():
    """kind -> (scene name, raw0 [N, 128] on the CPU).  "ties": pav_a's raw0 rounded to multiples of 1/16, with 37 rows of
    pav_b's appended (N = 640 037: a partial last tile of 64 rays)."""
    out = {k: (FRAMES[k][0], _with_extreme_rows(_frame_raw0(k))) for k in FRAMES}
    rounded = torch.round(torch.cat([out["pav_a"][1], out["pav_b"][1][:37]]) * 16) / 16
    out["ties"] = ("pavillon", rounded)
    return out


def _bulk_sorted(raw0):
    """The rows _with_extreme_rows left alone, each sorted descending."""
    r = torch.arange(raw0.shape[0])
    return torch.sort(raw0[(r % 32 != 5) & (r % 32 != 21)], dim=1, descending=True).values


def _thresholds(srt, K):
    """Two thresholds that are raw0 values (so some cells sit exactly on them): the median over rays of the K-th largest
    value and of the max(K // 2, 1)-th largest (srt = _bulk_sorted(raw0)); never <= 0 (the adaptive path)."""
    out = []
    for j in (K, max(K // 2, 1)):
        col = srt[:, j - 1]
        t = F32(torch.kthvalue(col, col.shape[0] // 2 + 1).values.item())
        if not t > 0:
            t = F32(2.0 ** -6)
        if out and t == out[0]:
            t = np.nextafter(t, F32(np.inf), dtype=F32)
        out.append(float(t))
    return out


@pytest.mark.parametrize("kind", ["pav_a", "pav_b", "shaped", "rand", "ndc", "ties"])
def test_stage2_whole_frame_bit_exact(frames, kind):
    """Every K in KS (thread kernel K <= 16, warp kernel above) at two thresholds each: count, offset, total, ray, cell,
    zp and z = zlut[cell], bit for bit.  Every case holds rays with no cell >= thr (the arg-max fallback), with 1..K and
    with more than K (except K = 128, where a ray cannot have more).  At K = 8 and 16 a raw0 that is only 4-byte aligned
    (served by the warp kernel) gives the aligned result."""
    scene_name, raw0 = frames[kind]
    scene = SCENES[scene_name]
    r = _renderer(scene)
    lut = se.zlut(scene)
    n = raw0.shape[0]
    dev = raw0.cuda()
    shifted = torch.empty(n * 128 + 1, dtype=torch.float32, device="cuda")[1:].view(n, 128)
    shifted.copy_(dev)
    assert shifted.data_ptr() % 16 == 4
    srt = _bulk_sorted(raw0)
    for K in KS:
        for thr in _thresholds(srt, K):
            what = f"{kind} K={K} thr={thr!r}"
            above = (raw0 >= thr).sum(1)
            assert bool((above == 0).any()) and bool(((above >= 1) & (above <= K)).any()), what
            assert K == 128 or bool((above > K).any()), what
            s2 = check_stage2(r, dev, raw0, thr, K, lut, what)
            if K in (8, 16):
                s2m = r.stage2(shifted, thr, K)
                for k in ("count", "offset", "cell", "ray", "z", "zp"):
                    assert torch.equal(s2m[k], s2[k]), (what, k)
    if kind == "ties":
        assert n % 64 == 37 and (raw0 * 16 == torch.round(raw0 * 16)).all()
    r.close()


# ------------------------------------------------------------------------------------------------ depth tables
@pytest.mark.parametrize("name", list(SCENES))
def test_adaptive_depth_table(name):
    """Rows that select all 128 cells read the whole adaptive table: z == zlut(scene) bit for bit."""
    scene = SCENES[name]
    r = _renderer(scene)
    s2 = r.stage2(torch.ones(3, 128, device="cuda"), 0.5, 128)
    assert s2["total"] == 3 * 128
    np.testing.assert_array_equal(s2["cell"].cpu().numpy(), np.tile(np.arange(128), 3))
    np.testing.assert_array_equal(_bits(s2["z"].cpu().numpy()), _bits(np.tile(se.zlut(scene), 3)))
    r.close()


@pytest.mark.parametrize("name", list(SCENES))
def test_dense_depth_table(name):
    """A dense render (thr 0, K 128) reports z_vals == zlut_dense(scene, 128) on every row, bit for bit."""
    scene = SCENES[name]
    sd0, sd1 = _weights(name)
    r = _renderer(scene, sd0, sd1)
    pose = np.asarray(scene["view_cell_center"], F32) + F32(0.05)
    dirs = r.generate_ray_directions(W, H)[::997]
    out = r.render_rays(pose, orc.rotation_yaw(20.0), dirs, 0.0, 128, want_aux=("z_vals",))
    z = out["z_vals"].cpu().numpy()
    assert z.shape == (dirs.shape[0], 128)
    np.testing.assert_array_equal(_bits(z), np.broadcast_to(_bits(se.zlut_dense(scene, 128)), z.shape))
    r.close()


# ---------------------------------------------------------------------------------------------- launch sequences
# (context, N, K, kind): "s2" = stage 2 at the call's threshold, "budget" = budget_threshold, "render" = render_rays.
# N is not monotone; K covers the K <= 8 and K <= 16 thread kernels and the warp kernel; context "B" is a second context
# on the same device, used in alternation with "A".
SEQUENCE = [("A", 640000, 8, "s2"), ("A", 1, 1, "s2"), ("B", 65, 17, "s2"), ("A", 4097, 16, "s2"), ("A", 4097, 8, "budget"),
            ("B", 63, 128, "s2"), ("A", 64, 9, "s2"), ("A", 0, 0, "render"), ("B", 640000, 100, "s2"), ("A", 1, 32, "s2"),
            ("A", 65, 17, "budget"), ("B", 4097, 2, "s2"), ("A", 65, 8, "s2"), ("A", 640000, 16, "s2"), ("B", 64, 128, "s2"),
            ("A", 63, 1, "s2"), ("B", 640000, 16, "budget"), ("A", 4097, 32, "s2"), ("B", 1, 128, "s2"), ("A", 64, 16, "s2"),
            ("A", 63, 8, "s2"), ("B", 65, 9, "s2"), ("A", 0, 0, "render"), ("A", 4097, 127, "s2"), ("B", 64, 8, "s2"),
            ("A", 1, 16, "s2"), ("A", 65, 100, "s2"), ("B", 4097, 17, "budget"), ("B", 63, 16, "s2"), ("A", 64, 2, "s2")]


def test_stage2_launch_sequence():
    """Fresh random raw0 on every call, so a tile state or ticket left over from an earlier launch (another size, another
    K, another kernel, a budget selection or a render in between) would show as a wrong offset or total."""
    sd0, sd1 = orc.make_weights("shaped", seed=0)
    ctx = {"A": _renderer(orc.SCENE_BARBERSHOP, sd0, sd1), "B": _renderer(orc.SCENE_PAVILLON)}
    lut = {"A": se.zlut(orc.SCENE_BARBERSHOP), "B": se.zlut(orc.SCENE_PAVILLON)}
    pose = np.asarray(orc.SCENE_BARBERSHOP["view_cell_center"], F32)
    dirs = ctx["A"].generate_ray_directions(W, H)[::21]
    ctx["A"].set_option("chunk_rays", 4096)                 # the render runs stage 2 once per 4096-ray chunk
    base = ctx["A"].render_rays(pose, orc.rotation_yaw(0.0), dirs, 0.2, 8)
    for i, (c, n, K, op) in enumerate(SEQUENCE):
        what = f"call {i}: {c} {op} N={n} K={K}"
        if op == "render":
            again = ctx[c].render_rays(pose, orc.rotation_yaw(0.0), dirs, 0.2, 8)
            assert torch.equal(again["rgb"], base["rgb"]) and torch.equal(again["n_samples"], base["n_samples"]), what
            continue
        g = torch.Generator().manual_seed(1000 + i)
        raw0 = torch.rand(n, 128, generator=g) * 1.2 - 0.8
        thr = (0.2, 0.05, 0.35)[i % 3]
        if op == "budget":
            B = n + (n * (K - 1)) // 3
            got = ctx[c].budget_threshold(raw0.cuda(), thr, K, B).item()
            assert _bits(got) == _bits(budget_threshold(raw0, thr, K, B)), what
        else:
            check_stage2(ctx[c], raw0.cuda(), raw0, thr, K, lut[c], what)
    for r in ctx.values():
        r.close()


# ------------------------------------------------------------------------------------- budget select, adversarial
N_BUDGET = 1_000_001        # odd: N (K - 1) is not a multiple of 4 for K = 2, 16, 128


def _from_bits(b):
    return np.asarray(b, np.uint32).view(F32)


def _budget_raw0(kind, seed):
    """[N_BUDGET, 128] rows of -1 with ~5 % of the cells candidates drawn from a small pool (long tie runs):
      spread  -- multiples of 2^-8 in [0.25, 4): many top-11-bit bins, round 0 decides;
      bin_r1  -- 1 + j 2^-13 (j < 64): one top-11-bit bin, round 1 decides;
      bin_r2  -- 1 + j 2^-23 (j < 16, values a few ulp apart): one top-21-bit prefix, round 2 decides;
      denormal -- k 2^-149 (k < 40) around the denormal thr_min 3 2^-149."""
    rng = np.random.default_rng(seed)
    if kind == "spread":
        pool = (np.arange(64, 1024) / 256.0).astype(F32)
    elif kind == "bin_r1":
        pool = _from_bits(0x3F800000 + (np.arange(64, dtype=np.uint32) << 10))
    elif kind == "bin_r2":
        pool = _from_bits(0x3F800000 + np.arange(16, dtype=np.uint32))
    else:
        pool = _from_bits(np.arange(1, 40, dtype=np.uint32))
    raw = np.full((N_BUDGET, 128), -1.0, F32)
    mask = rng.random((N_BUDGET, 128)) < 0.05
    raw[mask] = pool[rng.integers(0, pool.size, int(mask.sum()))]
    return raw


def _candidates_desc(raw, thr_min, K):
    v = -np.sort(-raw, axis=1)[:, 1:K]
    return np.sort(v[v >= F32(thr_min)])[::-1]


def _budgets(s, n):
    """B = N, N + 1, N + |S| - 1, N + |S|, N + |S| + 1, and two on a tie: the rank sought inside the longest run of equal
    candidates, and at its first element."""
    out = {"N": n, "N+1": n + 1, "N+|S|-1": n + s.size - 1, "N+|S|": n + s.size, "N+|S|+1": n + s.size + 1}
    if s.size > 1:
        starts = np.concatenate([[0], np.nonzero(s[1:] != s[:-1])[0] + 1])
        lens = np.diff(np.concatenate([starts, [s.size]]))
        i = int(np.argmax(lens))
        assert lens[i] >= 2
        out["tie_mid"] = n + int(starts[i] + lens[i] // 2)
        out["tie_first"] = n + int(starts[i])
    return out


def _check_budget(r, dev, raw, thr_min, K, B, what):
    """Device t* == budget_threshold bit for bit; stage 2 at t* keeps M <= B, one ulp below t* it exceeds B."""
    t = F32(r.budget_threshold(dev, thr_min, K, B).item())
    want = budget_threshold(raw, thr_min, K, B)
    assert _bits(t) == _bits(want), (what, B, float(t), float(want))
    m = r.stage2(dev, float(t), K)["total"]
    assert m <= B, (what, B, m)
    if t != F32(thr_min):
        below = np.nextafter(t, F32(-np.inf), dtype=F32)
        assert r.stage2(dev, float(below), K)["total"] > B, (what, B)
    return t


@pytest.fixture(scope="module")
def bare():
    r = _renderer(orc.SCENE_BARBERSHOP)
    yield r
    r.close()


@pytest.mark.parametrize("kind", ["spread", "bin_r1", "bin_r2", "denormal"])
def test_budget_select_adversarial(bare, kind):
    thr_min = 3 * 2.0 ** -149 if kind == "denormal" else 0.25
    raw = _budget_raw0(kind, seed=len(kind))
    dev = torch.from_numpy(raw).cuda()
    for K in (2, 16, 17, 128):
        s = _candidates_desc(raw, thr_min, K)
        assert s.size > 1000, (kind, K)
        if kind in ("bin_r1", "bin_r2", "denormal"):      # every candidate in one top-11-bit bin
            assert np.unique(_bits(s) >> 21).size == 1, (kind, K)
        if kind == "bin_r2":
            assert np.unique(_bits(s) >> 10).size == 1, (kind, K)
        ts = {label: _check_budget(bare, dev, raw, thr_min, K, B, f"{kind} K={K} {label}")
              for label, B in _budgets(s, N_BUDGET).items()}
        assert ts["N+|S|"] == F32(thr_min) and ts["N+|S|-1"] > F32(thr_min)


def test_budget_select_reads_the_last_keys(bare):
    """N (K - 1) = 1 or 3 (mod 4): the last 1 or 3 keys, the last ray's smallest candidates, are read only by the
    remainder of budget_hist_kernel's vector loop.  Every other key shares their top 21 bits (round 2 decides), and the rank
    sought is each of those last keys in turn."""
    thr_min = 0.25
    for K in (2, 16, 128):
        rng = np.random.default_rng(K)
        raw = np.full((N_BUDGET, 128), -1.0, F32)
        mask = rng.random((N_BUDGET, 128)) < 0.05
        raw[mask] = _from_bits(0x3F800000 + 2 * rng.integers(0, 500, int(mask.sum())).astype(np.uint32))   # even bits
        raw[-1] = -1.0
        raw[-1, 0] = 2.0                                                       # rank 1: not a key
        raw[-1, 1:K] = _from_bits(0x3F800000 + 999 - 2 * np.arange(K - 1, dtype=np.uint32))   # odd, descending by cell
        n_keys = N_BUDGET * (K - 1)
        tail = n_keys & 3
        assert tail in (1, 3)
        s = _candidates_desc(raw, thr_min, K)
        dev = torch.from_numpy(raw).cuda()
        # the last keys written: the thread kernels (K <= 16) write a ray's keys in pop order, so its smallest; the warp
        # kernel writes them in lane order per quarter j = cell % 4, so cells 119, 123 and 127 (the smallest of quarter 3)
        last = [119, 123, 127] if K > 16 else list(range(K - tail, K))
        for v in raw[-1, last]:
            q = int((s > v).sum())
            assert s[q] == v and (s == v).sum() == 1
            t = _check_budget(bare, dev, raw, thr_min, K, N_BUDGET + q, f"tail K={K}")
            assert t == np.nextafter(v, F32(np.inf), dtype=F32)


# ----------------------------------------------------------------------------------- budget renders, many chunks
@pytest.mark.parametrize("K,per_ray", [(8, 3), (32, 10)])
def test_budget_render_over_many_chunks(K, per_ray):
    """An 801x600 camera frame in chunks of 51 whole rows (40 851 rays, not a multiple of 64: 12 chunks, the last one
    short), through the camera entry and through the rays entry with the caller's d_oracle_weights: the budgeted render
    equals the fixed-threshold render at t*, and t* is budget_threshold of the frame's raw0."""
    sd0, sd1 = load_pavillon_weights()
    r = _renderer(orc.SCENE_PAVILLON, sd0, sd1)
    fw, fh = 801, 600
    n = fw * fh
    pose = np.asarray(orc.SCENE_PAVILLON["view_cell_center"], F32) + np.asarray([0.05, -0.03, 0.02], F32)
    rot = orc.rotation_yaw(60.0)
    thr_min, B = 0.05, per_ray * n
    r.set_option("chunk_rays", 50 * fw)                  # rounded up to whole rows: 51 rows per chunk
    r.set_option("sample_budget", B)
    cam = r.render_camera(pose, rot, fw, fh, thr_min, K, want_nsamples=True)
    t_cam = r.last_threshold()
    dirs = r.generate_ray_directions(fw, fh)
    rays = r.render_rays(pose, rot, dirs, thr_min, K, want_oracle_weights=True)
    t_rays = r.last_threshold()
    r.set_option("sample_budget", 0)
    fixed = r.render_camera(pose, rot, fw, fh, t_cam, K, want_nsamples=True)
    fixed_rays = r.render_rays(pose, rot, dirs, t_cam, K)
    r.close()
    want = budget_threshold(rays["oracle_weights"].cpu(), thr_min, K, B)
    assert _bits(t_cam) == _bits(want) and _bits(t_rays) == _bits(want)
    m = int(cam["n_samples"].long().sum())
    print(f"801x600 K={K}: t* = {t_cam:.6f}, M = {m} <= B = {B}")
    assert F32(thr_min) < t_cam and m <= B
    assert torch.equal(cam["rgb"], fixed["rgb"]) and torch.equal(cam["n_samples"], fixed["n_samples"])
    assert torch.equal(rays["rgb"], fixed_rays["rgb"]) and torch.equal(rays["n_samples"], fixed_rays["n_samples"])
    assert torch.equal(rays["rgb"], cam["rgb"])
