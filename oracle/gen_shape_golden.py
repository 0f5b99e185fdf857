"""TEST INFRASTRUCTURE -- golden fixtures of networks other than 8 x 256, from the UNMODIFIED reference
(/root/reference/src through oracle/ref_harness.py, CPU, build container only).

    python oracle/gen_shape_golden.py      # writes tests/golden/shape_*.npz, leaves the other fixtures alone

Each case builds the reference's models from `layers` / `layerWidth` / `skips` (ModelSelection.getModel,
src/models.py:363-372), loads `shape_oracle.make_shape_weights` into them and records one inference call, like
oracle/gen_golden.py's stage cases.  meta["weights"] holds the make_shape_weights arguments that rebuild the weights.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import adanerf_oracle as orc      # noqa: E402
from oracle import ref_harness as rh          # noqa: E402
from oracle import shape_oracle as so         # noqa: E402
from oracle.gen_golden import meta, save      # noqa: E402

# name: (layers, layerWidth, skips of the shading net, K, thr)
CASES = {
    "shape_6x128_s3_k8_t0.2": ((6, 6), (128, 128), "3", 8, 0.2),
    "shape_4x256_auto_k16_t0.15": ((4, 4), (256, 256), "auto", 16, 0.15),      # auto with D <= 4: no skip
    "shape_10x256_auto_k8_t0.2": ((8, 10), (256, 256), "auto", 8, 0.2),        # the largest side-parameter set
}


def shape_case(name, layers, widths, skip, K, thr, n_rays=256, stride=2503, w=800, h=800):
    scene = orc.SCENE_BARBERSHOP
    weights = dict(layers=list(layers), widths=list(widths), skip=skip, seed=0, thr=thr)
    sd0, sd1 = so.make_shape_weights(**weights)
    dirs_all = torch.from_numpy(rh.generate_ray_directions(
        w, h, scene["fov"], 0.5 * w / np.tan(0.5 * scene["fov"])).reshape(-1, 3)).float()
    pix = (torch.arange(n_rays) * stride) % (w * h)
    dirs = dirs_all[pix]
    pose = torch.tensor(scene["view_cell_center"], dtype=torch.float32)
    rot = orc.rotation_yaw(30.0)
    r = so.RefRenderer(scene, K=K, thr=thr, w=w, h=h, layers=layers, layerWidth=widths, skips=("", skip))
    r.load_state_dicts(sd0, sd1)
    st = r.stages(pose, rot, dirs)
    z = st["z_nan"]
    cnt = np.isfinite(z).sum(1)
    print(f"  {name}: mean spr {cnt.mean():.2f} hist {np.bincount(cnt, minlength=K + 1).tolist()}")
    save(name + ".npz", meta=meta(case=name, scene="barbershop", K=K, thr=thr, w=w, h=h, scene_params=scene, weights=weights,
                                  generator_shapes="oracle/gen_shape_golden.py"),
         pix=pix.numpy().astype(np.int64), dirs=dirs.numpy(), pose=pose.numpy(), rot=rot.numpy(),
         x0=st["x0"], raw0=st["raw0"], ray_o=st["ray_o"], ray_d=st["ray_d"], rgb=st["rgb"], weights=st["weights"],
         alpha=st["alpha"], depth_est=st["depth_est"], z_nan=z, asp=st["asp"], raw1_pad=st["raw1_pad"])


def main():
    torch.set_num_threads(8)
    for name, (layers, widths, skip, K, thr) in CASES.items():
        shape_case(name, layers, widths, skip, K, thr)


if __name__ == "__main__":
    main()
