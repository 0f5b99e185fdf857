"""Budget groups: several contexts, each rendering one row band of a frame, choose ONE sample-budget threshold -- the one a
single context would choose over the whole frame -- by summing the selection's histograms before every select round
(adn_set_budget_group, Renderer.set_budget_group, render_frame_distributed(sample_budget=), adn_multi "sample_budget").
The bands of a budgeted frame then equal the single-context budgeted frame bit for bit.

Every wait between members has a timeout: a member that never reaches a reduction fails the test instead of hanging it."""
import ctypes as C
import os
import re
import socket
import subprocess
import threading

import numpy as np
import pytest
import torch

from conftest import ROOT, load_pavillon_weights
from oracle import adanerf_oracle as orc
from test_sample_budget_oracle import budget_threshold

TIMEOUT = 120          # seconds any member waits for the others
SCENE = orc.SCENE_PAVILLON
THR = 0.05             # the floor threshold


def _bits(t):
    return np.float32(t).view(np.uint32)


def _view():
    pose = torch.tensor(SCENE["view_cell_center"]) + torch.tensor([0.05, -0.03, 0.02])
    rot = torch.tensor([[1, 0, 0], [0, 0, -1], [0, 1, 0]], dtype=torch.float32)
    return pose, rot


# ---- without a GPU -------------------------------------------------------------------------------------------------------
def test_group_symbols_are_exported_with_their_signatures():
    import __graft_entry__ as g
    g.build()
    from adanerf_b200 import _lib
    from adanerf_b200.multi import load_multi_library
    hdr = open(os.path.join(ROOT, "include", "adanerf_b200.h")).read()
    assert re.search(r"typedef int \(\*adn_budget_reduce_fn\)\(void\* user, uint64_t\* d_words, int64_t n_words, void\* stream\);", hdr)
    assert "adn_status adn_set_budget_group(adn_ctx* ctx, adn_budget_reduce_fn fn, void* user);" in hdr
    assert hasattr(C.CDLL(g.LIB), "adn_set_budget_group")
    lib = _lib.load_library()
    assert lib.adn_set_budget_group.argtypes == [C.c_void_p, _lib.BUDGET_REDUCE_FN, C.c_void_p]
    assert _lib.BUDGET_REDUCE_FN._restype_ is C.c_int
    assert _lib.BUDGET_REDUCE_FN._argtypes_ == (C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p)
    mhdr = open(os.path.join(ROOT, "include", "adanerf_b200_multi.h")).read()
    assert "adn_status adn_multi_last_threshold(adn_multi* m, float* thr_out);" in mhdr
    assert "adn_status adn_multi_last_samples(adn_multi* m, int64_t* band_samples);" in mhdr
    mlib = load_multi_library()
    assert mlib.adn_multi_last_threshold.argtypes == [C.c_void_p, C.POINTER(C.c_float)]
    assert mlib.adn_multi_last_samples.argtypes == [C.c_void_p, C.POINTER(C.c_int64)]
    raw = C.CDLL(g.MULTI_LIB)
    assert hasattr(raw, "adn_multi_last_threshold") and hasattr(raw, "adn_multi_last_samples")


def test_viewer_takes_gpus_with_budget(tmp_path):
    """-g N --budget B is a valid command line: it gets past argument parsing to loading the model on N devices."""
    import __graft_entry__ as g
    from adanerf_b200 import onnx_weights as ow
    g.build()
    sd0, sd1 = orc.make_weights("shaped", seed=0)
    d = tmp_path / "export"
    ow.write_export_dir(str(d), orc.SCENE_BARBERSHOP, sd0, sd1, 0.2, 8)
    r = subprocess.run([g.VIEWER, str(d), "-s", "64", "48", "-f", "1", "-g", "2", "--budget", str(64 * 48 * 3)], capture_output=True,
                       text=True, timeout=300)
    assert r.returncode != 2 and "usage" not in r.stderr and "renders on one device" not in r.stderr, r.stdout + r.stderr
    assert "K = 8" in r.stdout


# ---- one GPU: members in one process -------------------------------------------------------------------------------------
class HostSum:
    """Reducer of an in-process group: each member synchronises its stream, the words are summed on the host in member
    order and written back on the member's stream."""

    def __init__(self, n):
        self.barrier = threading.Barrier(n, timeout=TIMEOUT)
        self.words = [None] * n
        self.rounds = [0] * n

    def reducer(self, i):
        def fn(t):
            assert t.dtype == torch.int64 and t.numel() in (2049, 2048)
            torch.cuda.current_stream().synchronize()
            self.words[i] = t.cpu()
            self.barrier.wait()
            total = self.words[0].clone()
            for w in self.words[1:]:
                total += w
            self.barrier.wait()          # everyone has read every member's words before a next round replaces them
            t.copy_(total.to(t.device))
            self.rounds[i] += 1
        return fn


def _run(fns):
    """fns[i]() on a thread and a stream of its own each; their results, or the first exception re-raised."""
    n = len(fns)
    outs, errs = [None] * n, [None] * n
    streams = [torch.cuda.Stream() for _ in range(n)]

    def run(i):
        try:
            with torch.cuda.stream(streams[i]):
                outs[i] = fns[i]()
            streams[i].synchronize()
        except BaseException as e:      # noqa: BLE001 -- re-raised below
            errs[i] = e

    threads = [threading.Thread(target=run, args=(i,), daemon=True) for i in range(n)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=3 * TIMEOUT)
    assert not any(t.is_alive() for t in threads), "a member did not finish"
    for e in errs:
        if e is not None:
            raise e
    return outs


@pytest.fixture
def pav():
    from adanerf_b200 import Renderer
    sd0, sd1 = load_pavillon_weights()
    made = []

    def make(n=1):
        rs = [Renderer(SCENE, device=0, sampling_net=sd0, shading_net=sd1) for _ in range(n)]
        made.extend(rs)
        return rs
    yield make
    for r in made:
        r.close()


def _fixed_samples(make, W, H, K):
    """M of the fixed-threshold frame at the floor."""
    pose, rot = _view()
    return int(make()[0].render_camera(pose, rot, W, H, THR, K, want_nsamples=True)["n_samples"].long().sum())


def _single_budgeted(make, W, H, K, B):
    ref = make()[0]
    pose, rot = _view()
    ref.set_option("sample_budget", B)
    out = ref.render_camera(pose, rot, W, H, THR, K, want_nsamples=True)
    return out["rgb"], out["n_samples"], ref.last_threshold()


def _members(make, n, B, chunk_rays=()):
    rs = make(n)
    hs = HostSum(n)
    for i, r in enumerate(rs):
        r.set_option("sample_budget", B)
        r.set_budget_group(hs.reducer(i))
    for i, c in chunk_rays:
        rs[i].set_option("chunk_rays", c)
    return rs, hs


CASES = {
    # name: (K, whether B binds, rows of each band, (member, chunk_rays) pairs)
    "k8_two_equal_bands": (8, True, [400, 400], ()),
    "k16_uneven_bands_chunked": (16, True, [90, 510, 200], [(1, 40000)]),
    "k32_zero_row_member": (32, True, [300, 0, 250, 250], ()),
    "k16_budget_never_binds": (16, False, [500, 300], ()),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(CASES))
def test_bands_in_a_group_equal_the_single_context_frame(pav, case):
    K, binds, rows, chunks = CASES[case]
    W, H = 800, sum(rows)
    n = W * H
    m_thr = _fixed_samples(pav, W, H, K)
    assert m_thr > n
    B = (n + m_thr) // 2 if binds else m_thr                 # halfway between one sample per ray and the floor's M, or M(floor)
    rgb, ns, t_ref = _single_budgeted(pav, W, H, K, B)
    members, hs = _members(pav, len(rows), B, chunks)
    pose, rot = _view()
    row0 = np.cumsum([0] + rows[:-1])
    outs = _run([lambda r=r, a=int(a), b=b: r.render_camera(pose, rot, W, H, THR, K, row0=a, rows=b, want_nsamples=True)
                 for r, a, b in zip(members, row0, rows)])
    got_rgb = torch.cat([o["rgb"] for o in outs])
    got_ns = torch.cat([o["n_samples"] for o in outs])
    m = int(got_ns.long().sum())
    print(f"{case}: t* = {t_ref:.7g}, M = {m} <= B = {B}")
    assert hs.rounds == [3] * len(rows)                      # every member joined all three rounds, the empty one too
    for r in members:
        assert _bits(r.last_threshold()) == _bits(t_ref)
    if not binds:
        assert _bits(t_ref) == _bits(THR)
    else:
        assert t_ref > np.float32(THR)
    assert m <= B
    assert torch.equal(got_rgb, rgb) and torch.equal(got_ns, ns)


@pytest.mark.gpu
@pytest.mark.parametrize("K", [8, 32])
def test_stage_entry_in_a_group_equals_the_whole_rows_and_the_oracle(pav, K):
    """adn_budget_threshold on each member's band of raw0 (one band empty) == on the concatenated rows == the oracle."""
    ref = pav()[0]
    pose, rot = _view()
    W, H = 800, 200
    fixed = ref.render_rays(pose, rot, ref.generate_ray_directions(W, H), THR, K, want_oracle_weights=True)
    raw0 = fixed["oracle_weights"]
    n = W * H
    B = (n + int(fixed["n_samples"].long().sum())) // 2
    whole = ref.budget_threshold(raw0, THR, K, B).item()
    want = budget_threshold(raw0.cpu(), THR, K, B)
    cuts = [0, 37_001, 37_001, 120_000, n]                   # bands of 37 001, 0, 82 999 and 40 000 rows
    members, hs = _members(pav, len(cuts) - 1, B)
    got = _run([lambda r=r, a=a, b=b: r.budget_threshold(raw0[a:b], THR, K, B).item()
                for r, a, b in zip(members, cuts[:-1], cuts[1:])])
    assert hs.rounds == [3] * len(members)
    assert _bits(whole) == _bits(want) and whole > np.float32(THR)
    for t in got:
        assert _bits(t) == _bits(whole)


@pytest.mark.gpu
def test_reducer_failure_fails_the_call_and_the_context_stays_usable(pav):
    from adanerf_b200 import AdnError
    W, H, K = 800, 100, 16
    B = W * H * 8
    rgb, ns, t_ref = _single_budgeted(pav, W, H, K, B)
    r = pav()[0]
    r.set_option("sample_budget", B)
    pose, rot = _view()
    calls = []

    def flaky(t):
        calls.append(t.numel())
        if len(calls) == 2:
            raise RuntimeError("link down")
    r.set_budget_group(flaky)                                   # a group of one: the sum is the member's own words
    with pytest.raises(AdnError, match="reducer returned 1 in select round 1") as e:
        r.render_camera(pose, rot, W, H, THR, K)
    assert isinstance(e.value.__cause__, RuntimeError)
    again = r.render_camera(pose, rot, W, H, THR, K, want_nsamples=True)
    assert calls == [2049, 2048, 2049, 2048, 2048]
    assert _bits(r.last_threshold()) == _bits(t_ref)
    assert torch.equal(again["rgb"], rgb) and torch.equal(again["n_samples"], ns)

    def broken(t):
        raise RuntimeError("must not be called")
    r.set_budget_group(broken)
    with pytest.raises(AdnError, match="round 0"):
        r.render_camera(pose, rot, W, H, THR, K)
    r.set_budget_group(None)                                    # per-context selection again: the reducer is not called
    alone = r.render_camera(pose, rot, W, H, THR, K, row0=30, rows=40, want_nsamples=True)
    solo = pav()[0]
    solo.set_option("sample_budget", B)
    want = solo.render_camera(pose, rot, W, H, THR, K, row0=30, rows=40, want_nsamples=True)
    assert _bits(r.last_threshold()) == _bits(solo.last_threshold())
    assert torch.equal(alone["rgb"], want["rgb"]) and torch.equal(alone["n_samples"], want["n_samples"])


@pytest.mark.gpu
def test_multi_budget_is_checked_against_the_frame(pav):
    """adn_multi on one device: B < W * H is refused before anything is enqueued; a frame within the budget equals the
    single-context budgeted frame and reports its threshold and M."""
    from adanerf_b200 import AdnError
    from adanerf_b200.multi import MultiRenderer
    sd0, sd1 = load_pavillon_weights()
    W, H, K = 800, 300, 16
    B = W * H * 8
    rgb, ns, t_ref = _single_budgeted(pav, W, H, K, B)
    m = MultiRenderer(SCENE, [0], sd0, sd1)
    try:
        pose, rot = _view()
        m.set_option("sample_budget", W * H - 1)
        with pytest.raises(AdnError, match="below the 240000 rays of the frame"):
            m.render_camera(pose, rot, W, H, THR, K)
        with pytest.raises(AdnError, match="no frame in flight"):
            m.wait_frame()                                          # nothing was enqueued
        m.set_option("sample_budget", B)
        m.render_camera(pose, rot, W, H, THR, K)
        assert torch.equal(m.wait_frame().cpu(), rgb.cpu())
        assert _bits(m.last_threshold()) == _bits(t_ref)
        assert m.last_samples() == [int(ns.long().sum())]
    finally:
        m.close()


# ---- one GPU: two processes, torch.distributed -------------------------------------------------------------------------
def _dist_worker(rank, world, port, q):
    import datetime
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=TIMEOUT))
    try:
        from adanerf_b200 import Renderer
        from adanerf_b200.tiling import render_frame_distributed
        sd0, sd1 = load_pavillon_weights()
        r = Renderer(SCENE, device=0, sampling_net=sd0, shading_net=sd1)
        pose, rot = _view()
        W, H, K = 800, 601, 16
        B = W * H * 8
        try:
            render_frame_distributed(r, pose, rot, W, H, THR, K, dst=0, sample_budget=W * H - 1)
            refused = False
        except ValueError as e:
            refused = "below" in str(e)
        full = render_frame_distributed(r, pose, rot, W, H, THR, K, dst=0, sample_budget=B)
        t = r.last_threshold()
        res = dict(rank=rank, refused=refused, t=float(t))
        if rank == 0:
            ref = Renderer(SCENE, device=0, sampling_net=sd0, shading_net=sd1)
            ref.set_option("sample_budget", B)
            want = ref.render_camera(pose, rot, W, H, THR, K)["rgb"]
            res.update(equal=bool(torch.equal(full, want)), t_ref=float(ref.last_threshold()))
            ref.close()
        r.close()
        q.put(res)
    except BaseException as e:          # noqa: BLE001 -- reported to the test
        q.put(dict(rank=rank, error=repr(e)))
    finally:
        dist.destroy_process_group()


@pytest.mark.gpu
def test_render_frame_distributed_with_a_budget_world2_on_one_gpu():
    """Two gloo ranks on cuda:0, uneven bands (601 rows): the frame gathered on rank 0 equals the single-context budgeted
    frame bit for bit, both ranks report its threshold, and B < W * H is refused on both ranks before anything runs."""
    import torch.multiprocessing as mp
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_dist_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    try:
        res = sorted((q.get(timeout=4 * TIMEOUT) for _ in procs), key=lambda d: d["rank"])
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.terminate()
                p.join(timeout=30)
    assert all("error" not in d for d in res), res
    assert all(d["refused"] for d in res), res
    assert res[0]["equal"], res
    assert _bits(res[0]["t"]) == _bits(res[0]["t_ref"]) == _bits(res[1]["t"]) and res[0]["t_ref"] > np.float32(THR)


# ---- two or more GPUs --------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
@pytest.mark.parametrize("H", [800, 203])
def test_multi_budgeted_frame_equals_the_single_gpu_frame(pav, H):
    from adanerf_b200.multi import MultiRenderer
    sd0, sd1 = load_pavillon_weights()
    W, K = 800, 16
    B = W * H * 8
    rgb, ns, t_ref = _single_budgeted(pav, W, H, K, B)
    G = min(torch.cuda.device_count(), 4)
    m = MultiRenderer(SCENE, list(range(G)), sd0, sd1)
    try:
        m.set_option("sample_budget", B)
        pose, rot = _view()
        m.render_camera(pose, rot, W, H, THR, K)
        assert torch.equal(m.wait_frame().cpu(), rgb.cpu())
        assert _bits(m.last_threshold()) == _bits(t_ref)
        assert sum(m.last_samples()) == int(ns.long().sum()) <= B
    finally:
        m.close()


@pytest.mark.gpu
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_viewer_on_two_gpus_prints_the_one_gpu_thresholds(tmp_path):
    import __graft_entry__ as g
    from adanerf_b200 import onnx_weights as ow
    g.build()
    sd0, sd1 = orc.make_weights("shaped", seed=0)
    d = tmp_path / "export"
    ow.write_export_dir(str(d), orc.SCENE_BARBERSHOP, sd0, sd1, 0.2, 8)
    budget = 400 * 301 * 3
    pattern = r"frame (\d+): threshold ([0-9.e+-]+), (\d+) samples \(budget (\d+)\)"
    runs = {}
    for gpus in (1, 2):
        r = subprocess.run([g.VIEWER, str(d), "-s", "400", "301", "-f", "3", "-g", str(gpus), "--budget", str(budget)],
                           capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stdout + r.stderr
        runs[gpus] = re.findall(pattern, r.stdout)
        assert len(runs[gpus]) == 3, r.stdout
    for (f1, t1, m1, b1), (f2, t2, m2, b2) in zip(runs[1], runs[2]):
        assert f1 == f2 and t1 == t2 and m1 == m2, (runs[1], runs[2])
        assert int(m2) <= int(b2) == budget
