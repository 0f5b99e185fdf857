"""Multi-image inference on CPU: the live reference's TrainConfig.inference over a batch of two images equals the fixtures
tests/golden/views_*.npz bit for bit and equals its per-image calls concatenated (torch on one thread), and the adapter turns
an n_images = 2 batch of a live TrainConfig into one views call with image-major outputs."""
import os

import numpy as np
import pytest
import torch

from adanerf_b200.synthetic import load_npz
from oracle import ref_harness as rh
from oracle.gen_views_golden import CASES, N_RAYS, V, arrays, case_inputs, inference, reference

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
needs_ref = pytest.mark.skipif(not rh.available(), reason="reference checkout not present")


@pytest.fixture
def one_thread():
    n = torch.get_num_threads()
    torch.set_num_threads(1)
    yield
    torch.set_num_threads(n)


def test_fixtures_hold_two_differing_views():
    for i, name in enumerate(CASES):
        g = load_npz(os.path.join(GOLDEN, f"views_{name}.npz"))
        assert g["poses"].shape == (V, 3) and g["rots"].shape == (V, 3, 3) and g["dirs"].shape == (V, N_RAYS, 3)
        assert g["rgb"].shape == (V * N_RAYS, 3) and g["depth_est"].shape == (V * N_RAYS,)
        assert ("asp" in g) == (CASES[name][0] == 0)
        assert not np.array_equal(g["poses"][0], g["poses"][1]) and not np.array_equal(g["rots"][0], g["rots"][1])
        _, poses, rots, dirs, _, _ = case_inputs(name, 500 + i)
        for k, t in (("poses", poses), ("rots", rots), ("dirs", dirs)):
            np.testing.assert_array_equal(g[k], t.numpy(), err_msg=f"{name} {k}")


@needs_ref
@pytest.mark.parametrize("i,name", list(enumerate(CASES)))
def test_live_reference_multi_image_equals_fixture_and_per_image_calls(one_thread, i, name):
    seed = 500 + i
    g = load_npz(os.path.join(GOLDEN, f"views_{name}.npz"))
    _, poses, rots, dirs, _, _ = case_inputs(name, seed)
    ref = reference(name, seed)
    got = arrays(*inference(ref, poses, rots, dirs))
    for k, v in got.items():
        np.testing.assert_array_equal(v, g[k], err_msg=f"{name} {k} against the fixture")
    for v in range(V):
        one = arrays(*inference(ref, poses[v:v + 1], rots[v:v + 1], dirs[v:v + 1]))
        for k, a in one.items():
            part = got[k][v * N_RAYS:(v + 1) * N_RAYS]
            if CASES[name][0] == 0:
                np.testing.assert_array_equal(part, a, err_msg=f"{name} view {v} {k}")
            else:
                # nerf_raw2outputs' sums over the K samples of a [n, K] batch (samplers 1 and 2): ATen vectorises them
                # across rays, so a colour can differ from the one-image call in its last bits (SURVEY)
                np.testing.assert_allclose(part, a, rtol=0, atol=1e-7, err_msg=f"{name} view {v} {k}")


class _Recorder:
    """Stands in for the Renderer: records the call the adapter makes and returns outputs of the shapes it asks for."""

    def __init__(self):
        self.calls = []

    def _out(self, n, K, kw):
        out = dict(rgb=torch.zeros(n, 3), n_samples=torch.full((n,), K, dtype=torch.int32),
                   oracle_weights=torch.zeros(n, 128) if kw["want_oracle_weights"] else None)
        for k in kw["want_aux"] or ():
            out[k] = torch.zeros((n, K) if k in ("weights", "alpha", "z_vals") else (n,))
        return out

    def render_rays(self, pose, rot, dirs, thr, K, **kw):
        self.calls.append(("rays", tuple(pose.shape), tuple(rot.shape), tuple(dirs.shape)))
        return self._out(dirs.shape[0], K, kw)

    def render_views(self, poses, rots, dirs, thr, K, **kw):
        self.calls.append(("views", tuple(poses.shape), tuple(rots.shape), tuple(dirs.shape)))
        return self._out(dirs.shape[0] * dirs.shape[1], K, kw)


@needs_ref
def test_adapter_two_image_batch_from_live_train_config():
    """A SampleDataWrapper of two images from the live reference reaches the renderer as one views call, and the adapter
    returns the reference's flattened shapes."""
    from adanerf_b200.adapter import B200Inference, KEY_ASP, KEY_ORACLE, KEY_DEPTH
    name = "pav_k16"
    ref = reference(name, 500)
    ref.tc.dataset_info = ref.dataset_info          # what TrainConfig.initialize sets
    scene, models, thr, K = B200Inference.args_from_train_config(ref.tc)
    assert (thr, K) == (CASES[name][3], CASES[name][2])
    _, poses, rots, dirs, _, _ = case_inputs(name, 500)
    from datasets import SampleDataWrapper, DatasetKeyConstants as D
    d = {D.image_pose: poses, D.image_rotation: rots, D.ray_directions_samples: dirs}
    batch = SampleDataWrapper([dict(d), dict(d)], [], False)
    inf = B200Inference.__new__(B200Inference)
    inf.renderer, inf.threshold, inf.K, inf.sampler = _Recorder(), thr, K, 0
    inf.want_oracle_weights, inf.want_aux = True, True
    outs, dicts = inf.inference(batch)
    assert inf.renderer.calls == [("views", (V, 3), (V, 3, 3), (V, N_RAYS, 3))]
    n = V * N_RAYS
    assert outs[-1].shape == (n, 3) and dicts[1][KEY_ASP].shape == (n,) and dicts[1][KEY_ORACLE].shape == (n, 128)
    assert dicts[1][KEY_DEPTH].shape == (n, 1)
    inf.renderer.calls.clear()
    one = SampleDataWrapper([{k: v[:1] for k, v in d.items()}] * 2, [], False)
    inf.inference(one)
    assert inf.renderer.calls == [("rays", (3,), (3, 3), (N_RAYS, 3))]
