"""The sample-budget rule (budget_threshold, the exact CPU restatement the GPU tests compare the device selection with),
checked against the sampler it budgets (oracle.stage2_sample, the restatement of FromClassifiedDepthAdaptive.generate): the
chosen threshold t* keeps M(t*) <= B, and it is the smallest such fp32 threshold >= thr_min, on the golden raw0 sets
(stage2_stress holds exact ties)."""
import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import adanerf_oracle as orc

SETS = {"pav_k8_t0.2": 0.2, "pav_k16_t0.15": 0.15, "rand_k8_t0.2": 0.2, "stage2_stress": 0.2}
KS = [1, 8, 16, 32, 128]


def budget_threshold(raw0, thr_min, K, max_samples):
    """Sample budget: the smallest fp32 threshold t >= thr_min (> 0) at which stage2_sample yields at most max_samples
    samples in all.  For t > 0 the sampler gives ray r  n_r(t) = clamp(#{cells >= t}, 1, K)  samples
    (src/nerf_raymarch_common.py:726-749: sort descending, `>=`, cap at K, arg-max fallback), hence

        M(t) = N + #{(r, j) : 2 <= j <= K, v_r^(j) >= t},   v_r^(j) = the j-th largest raw0 value of ray r (ties counted).

    With S = the multiset of those rank-2..K values that are >= thr_min and Q = max_samples - N:
    |S| <= Q -> t = thr_min;  otherwise t = nextafterf(s_(Q+1), +inf), s_(Q+1) = the (Q+1)-th largest element of S.
    Returns a numpy float32."""
    v = np.asarray(raw0.numpy() if isinstance(raw0, torch.Tensor) else raw0, dtype=np.float32)
    n = v.shape[0]
    t0 = np.float32(thr_min)
    if not t0 > 0 or max_samples < n:
        raise ValueError("budget_threshold: need thr_min > 0 and max_samples >= N")
    ranked = -np.sort(-v, axis=1)[:, 1:K]          # rank 2..K of every ray, descending
    s = np.sort(ranked[ranked >= t0])[::-1]         # S, descending
    q = int(max_samples) - n
    if s.size <= q:
        return t0
    return np.nextafter(s[q], np.float32(np.inf), dtype=np.float32)


def _raw0(name):
    g = load_golden(name)
    dr = g["meta"].get("depth_range") or g["meta"]["scene_params"]["depth_range"]
    return torch.from_numpy(g["raw0"]), dr


def _samples(raw0, t, K, dr):
    return int(orc.stage2_sample(raw0, float(t), K, dr)["count"].sum())


def _candidates(raw0, thr_min, K):
    """S of the identity, descending: every ray's rank-2..K values >= thr_min."""
    v = -np.sort(-raw0.numpy(), axis=1)[:, 1:K]
    return np.sort(v[v >= np.float32(thr_min)])[::-1]


def budgets(raw0, thr_min, K):
    n = raw0.shape[0]
    s = _candidates(raw0, thr_min, K)
    out = {"one_per_ray": n, "n_times_k": n * K, "above_n_times_k": n * K + 7}
    for f in (0.1, 0.5, 0.9):
        out[f"mid{f}"] = n + int(f * s.size)
    run = np.nonzero(s[1:] == s[:-1])[0]   # s[i] == s[i + 1]: B = N + i + 1 makes s_(Q+1) a tied value
    if run.size:
        out["on_tie"] = n + int(run[run.size // 2]) + 1
    return out


@pytest.mark.parametrize("K", KS)
@pytest.mark.parametrize("name", sorted(SETS))
def test_budget_threshold_is_the_smallest_that_fits(name, K):
    raw0, dr = _raw0(name)
    thr_min = SETS[name]
    n = raw0.shape[0]
    for label, B in budgets(raw0, thr_min, K).items():
        t = budget_threshold(raw0, thr_min, K, B)
        assert t.dtype == np.float32 and t >= np.float32(thr_min), label
        m = _samples(raw0, t, K, dr)
        assert m <= B, (label, B, m)
        if t != np.float32(thr_min):
            prev = np.nextafter(t, np.float32(-np.inf), dtype=np.float32)
            assert _samples(raw0, prev, K, dr) > B, (label, B)
        if label == "one_per_ray":
            assert m == n
        if label in ("n_times_k", "above_n_times_k") or K == 1:
            assert t == np.float32(thr_min), label
        # the identity behind the rule: M(t) = N + #{rank-2..K values >= t}
        assert m == n + int((_candidates(raw0, thr_min, K) >= t).sum()), label


def test_stress_set_has_a_tie_at_the_budget():
    raw0, dr = _raw0("stage2_stress")
    B = budgets(raw0, 0.2, 16)["on_tie"]
    t = budget_threshold(raw0, 0.2, 16, B)
    s = _candidates(raw0, 0.2, 16)
    tied = s[B - raw0.shape[0]]
    assert (s == tied).sum() >= 2 and t == np.nextafter(tied, np.float32(np.inf), dtype=np.float32)
    assert _samples(raw0, t, 16, dr) < B          # the whole tie run is dropped: the budget is not met exactly


def test_budget_threshold_rejects_bad_arguments():
    raw0, _ = _raw0("pav_k8_t0.2")
    with pytest.raises(ValueError):
        budget_threshold(raw0, 0.0, 8, 10_000)
    with pytest.raises(ValueError):
        budget_threshold(raw0, 0.2, 8, raw0.shape[0] - 1)
