"""B200Inference.from_train_config against what an initialised reference TrainConfig carries (tests/golden/
live_train_config.json, recorded from the live reference by oracle/gen_live_golden.py): the attribute names it reads --
f_in[1].{depth_range, max_depth, z_near, z_far, z_sampler.threshold, n_ray_samples}, dataset_info.view.{view_cell_center,
view_cell_size, fov} (src/features.py:343-360, 747-767; src/train_data.py:60-110) -- and the values the renderer needs.
No GPU: only the extraction is exercised."""
import json
import os
from types import SimpleNamespace

import numpy as np
import pytest

from conftest import GOLDEN
from oracle import adanerf_oracle as orc

CONFIGS = json.load(open(os.path.join(GOLDEN, "live_train_config.json")))["configs"]


class _Model:
    def __init__(self, keys):
        self._keys = keys

    def state_dict(self):
        return {k: None for k in self._keys}


def _train_config(c):
    """An object with the recorded TrainConfig's attribute paths and values."""
    f = c["f_in1"]
    f1 = SimpleNamespace(depth_range=f["depth_range"], max_depth=f["max_depth"], z_near=f["z_near"], z_far=f["z_far"],
                         z_sampler=SimpleNamespace(threshold=f["z_sampler_threshold"]), n_ray_samples=f["n_ray_samples"],
                         useNDC=f["useNDC"])
    return SimpleNamespace(f_in=[SimpleNamespace(), f1], dataset_info=SimpleNamespace(view=SimpleNamespace(**c["view"])),
                           models=[_Model(c["state_dict_keys"][0]), _Model(c["state_dict_keys"][1])])


@pytest.mark.parametrize("K,thr", [(8, 0.2), (16, 0.15)])
def test_scene_and_sampler_fields_from_live_train_config(K, thr):
    from adanerf_b200.adapter import B200Inference
    scene = orc.SCENE_PAVILLON
    c = next(c for c in CONFIGS if c["K"] == K and c["thr"] == thr)
    tc = _train_config(c)
    got, models, got_thr, got_k = B200Inference.args_from_train_config(tc)
    assert got_k == K and abs(got_thr - thr) < 1e-7
    assert models[0] is tc.models[0] and models[1] is tc.models[1]
    np.testing.assert_allclose(got["view_cell_center"], scene["view_cell_center"], rtol=0, atol=0)
    np.testing.assert_allclose(got["view_cell_size"], scene["view_cell_size"], rtol=0, atol=0)
    np.testing.assert_allclose(got["depth_range"], scene["depth_range"], rtol=1e-7)    # the WARPED range (features.py:355)
    assert abs(got["max_depth"] - scene["max_depth"]) < 1e-6 * scene["max_depth"]
    assert abs(got["fov"] - scene["fov"]) < 1e-7
    assert got["z_near"] == pytest.approx(0.001) and got["z_far"] == pytest.approx(1.0)
    assert not got.get("use_ndc", False)
    # the state_dict names the packer expects (src/models.py:18-82, 200-250)
    assert "layers.7.weight" in tc.models[0].state_dict() and "pts_linears.5.weight" in tc.models[1].state_dict()
