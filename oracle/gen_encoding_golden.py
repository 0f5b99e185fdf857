"""TEST INFRASTRUCTURE -- golden fixtures of positional encodings other than posEncArgs 10-4 (2-2 for the NDC sampling
net), from the UNMODIFIED reference (/root/reference/src through oracle/ref_harness.py, CPU, build container only).

    python oracle/gen_encoding_golden.py      # writes tests/golden/enc_*.npz, leaves the other fixtures alone

Each case sets the reference's posEnc / posEncArgs (src/util/config.py:46-48; FeatureSet, src/features.py:326-339;
NeRF.input_ch, src/models.py:216-224) and the shading net's layers / layerWidth / skips, loads `case_weights` into the
models it builds and records one inference call, like oracle/gen_shape_golden.py.  `case_weights` needs no reference, so
the tests rebuild the weights from the case name.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import adanerf_oracle as orc      # noqa: E402
from oracle import ref_harness as rh          # noqa: E402

# name: (posEnc, posEncArgs, ndc, shading (layers, width, skips entry), K, thr) -- both shading blocks at their limit with a
# two-block position input through the skip consumer; the sampling format at its limit (126 columns); no encoding on
# either net; NDC with a two-block position input.
CASES = {
    "enc_s10-4_p20-10_k8_t0.2": (("nerf", "nerf"), ("10-4", "20-10"), False, (8, 256, "auto"), 8, 0.2),
    "enc_s16-4_p6-2_k16_t0.15": (("nerf", "nerf"), ("16-4", "6-2"), False, (8, 256, "auto"), 16, 0.15),
    "enc_none_6x128_s3_k8_t0.2": (("none", "none"), ("10-4", "10-4"), False, (6, 128, "3"), 8, 0.2),
    "enc_ndc_s2-2_p12-6_k16_t0.15": (("nerf", "nerf"), ("2-2", "12-6"), True, (8, 256, "auto"), 16, 0.15),
}


def bands(pos_enc, pos_enc_args):
    """[(P0, D0), (P, D)]: a net's band counts, (0, 0) for posEnc none (NoEncoding, the 3 inputs alone)."""
    return [(0, 0) if e == "none" else tuple(int(x) for x in a.split("-")) for e, a in zip(pos_enc, pos_enc_args)]


def case_scene(name):
    """The renderer's scene dict of a case (renderer.make_scene fields): -1 / -1 for posEnc none, and -1 for a literal 0 in
    the sampling net's fields (0 there means "the shading net's count")."""
    pos_enc, args, ndc, _, _, _ = CASES[name]
    (p0, d0), (p, d) = bands(pos_enc, args)
    scene = dict(orc.SCENE_BARBERSHOP)
    if pos_enc[1] == "none":
        p = d = -1
    if ndc:
        scene.update(use_ndc=True, w=800, h=800)
    return dict(scene, n_freq_pos=p, n_freq_dir=d, n_freq_pos0=p0 or -1, n_freq_dir0=d0 or -1)


def case_weights(name, seed=0, target_spr=None):
    """The case's networks (encoding_weights with the case's encodings, shading shape and thr; target K / 2 + 1)."""
    pos_enc, args, ndc, shape, K, thr = CASES[name]
    return encoding_weights(*bands(pos_enc, args), shape, thr, K / 2 + 1 if target_spr is None else target_spr,
                            case_scene(name), seed)


def encoding_weights(b0, b1, shape, thr, target_spr, scene, seed=0):
    """Networks for sampling bands b0 = (P0, D0) and shading bands b1 = (P, D), shading (layers, width, skips entry): the
    reference's init order (adanerf_oracle.init_*; BaseNet, NeRF with those input widths), then the sampling net's last
    layer scaled by 0.15 and its bias shifted until the mean number of cells >= thr is ~target_spr on a probe batch of
    `scene`, so that rays keep ragged 1..K samples."""
    (p0, d0), (p, d) = b0, b1
    D1, W1, skip = shape
    torch.manual_seed(seed)
    sd0 = orc.init_sampling_net(n_in=6 + 6 * (p0 + d0))
    sd1 = orc.init_shading_net(input_ch=3 + 6 * p, input_ch_views=3 + 6 * d, W=W1, D=D1,
                               skips=(4,) if skip == "auto" else (int(skip),))
    sd0["layers.7.weight"] = sd0["layers.7.weight"] * 0.15
    sd0["layers.7.bias"] = sd0["layers.7.bias"] * 0.15
    dirs = torch.from_numpy(orc.generate_ray_directions(800, 800, scene["fov"]).reshape(-1, 3)[::157]).float()
    x0, _, _ = orc.stage0_sphere_pos_dir(torch.tensor(scene["view_cell_center"], dtype=torch.float32), torch.eye(3), dirs,
                                         scene, n_freq_pos=p0, n_freq_dir=d0)
    with torch.no_grad():
        base = orc.mlp0_forward(x0, sd0)
    lo, hi = -4.0, 4.0
    for _ in range(40):
        mid = 0.5 * (lo + hi)
        if float(((base + mid) >= thr).sum(1).float().mean()) > target_spr:
            hi = mid
        else:
            lo = mid
    sd0["layers.7.bias"] = sd0["layers.7.bias"] + 0.5 * (lo + hi)
    return sd0, sd1


class RefRenderer(rh.RefRenderer):
    """ref_harness.RefRenderer with the case's posEnc / posEncArgs and shading-net shape (build container only)."""

    def __init__(self, name, w=800, h=800, seed=0):
        rh._install_stubs()
        torch.manual_seed(seed)
        from features import FeatureSet
        from models import ModelSelection
        from train_data import TrainConfig
        pos_enc, args, ndc, (D1, W1, skip), K, thr = CASES[name]
        scene = case_scene(name)
        self.cfg = rh.make_config(K=K, thr=thr, ndc=ndc)
        self.cfg.posEnc, self.cfg.posEncArgs = list(pos_enc), list(args)
        self.cfg.layers, self.cfg.layerWidth, self.cfg.skips = [8, D1], [256, W1], ["", skip]
        self.dataset_info = rh.make_dataset_info(scene, w, h, ndc=ndc)
        f_in, f_out = FeatureSet.get_sets(self.cfg, "cpu")
        for f in list(f_in) + list(f_out):
            f.initialize(self.cfg, self.dataset_info, "cpu")
        models = [ModelSelection.getModel(self.cfg, f_in[i].n_feat, 128 if i == 0 else 4, "cpu", i) for i in range(2)]
        tc = TrainConfig()
        tc.f_in, tc.f_out, tc.models, tc.config_file = f_in, f_out, models, self.cfg
        tc.device, tc.dataset_info = "cpu", self.dataset_info
        self.tc = tc


def case_rays(name, n_rays=256, stride=2503, w=800, h=800):
    """(pix, dirs, pose, rot) of a case: every stride-th pixel of the frame, the camera at the view-cell centre, yawed."""
    scene = case_scene(name)
    dirs_all = torch.from_numpy(rh.generate_ray_directions(
        w, h, scene["fov"], 0.5 * w / np.tan(0.5 * scene["fov"])).reshape(-1, 3)).float()
    pix = (torch.arange(n_rays) * stride) % (w * h)
    return pix, dirs_all[pix], torch.tensor(scene["view_cell_center"], dtype=torch.float32), orc.rotation_yaw(30.0)


def encoding_case(name, n_x1_rays=16):
    from oracle.gen_golden import meta, save
    pos_enc, args, ndc, shape, K, thr = CASES[name]
    pix, dirs, pose, rot = case_rays(name)
    r = RefRenderer(name)
    r.load_state_dicts(*case_weights(name))
    st = r.stages(pose, rot, dirs)
    z = st["z_nan"]
    cnt = np.isfinite(z).sum(1)
    print(f"  {name}: x0 {st['x0'].shape[1]} columns, x1 {st['x1_nan'].shape[2]}; mean spr {cnt.mean():.2f} "
          f"hist {np.bincount(cnt, minlength=K + 1).tolist()}")
    save(name + ".npz", meta=meta(case=name, K=K, thr=thr, w=800, h=800, scene_params=case_scene(name), pos_enc=list(pos_enc),
                                  pos_enc_args=list(args), shading=list(shape), generator_encodings="oracle/gen_encoding_golden.py"),
         pix=pix.numpy().astype(np.int64), dirs=dirs.numpy(), pose=pose.numpy(), rot=rot.numpy(),
         x0=st["x0"], raw0=st["raw0"], ray_o=st["ray_o"], ray_d=st["ray_d"], rgb=st["rgb"], weights=st["weights"],
         z_nan=z, asp=st["asp"], raw1_pad=st["raw1_pad"], x1_nan=st["x1_nan"][:n_x1_rays])


def main():
    torch.set_num_threads(8)
    for name in CASES:
        encoding_case(name)


if __name__ == "__main__":
    main()
