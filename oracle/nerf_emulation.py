"""fp32-FAITHFUL EMULATION OF THE PLAIN-NERF RAY KERNEL -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

`camera_rays_kernel` (adanerf_b200/csrc/stages.cu, option "sampler" = 2) restated operation for operation in numpy float32,
on top of oracle/stage_emulation.py's rotation and scene constants: tests/test_nerf_gpu.py compares it with
`assert_array_equal` on whole frames.  The kernel's depth table is stage_emulation.zlut_dense (the same host table).
"""
import numpy as np

from oracle.stage_emulation import F32, rotate, scene_constants


# ------------------------------------------------------------------------------------------- camera rays (sampler 2)
def camera_rays(pose, rot, dirs, scene):
    """camera_rays_kernel (stages.cu) -> (ray_o [N,3] = pose, ray_d [N,3] = R d as the FMA chain of `rotate`, ray_dirs
    [N,3]: ray_d, or on NDC scenes ndc_ray's un-normalised direction in sample_inputs' operation order)."""
    k = scene_constants(scene)
    pose = np.asarray(pose, F32).reshape(3)
    nds = rotate(rot, dirs)
    ray_o = np.broadcast_to(pose, nds.shape).copy()
    if not k["ndc"]:
        return ray_o, nds, nds.copy()
    cw, ch = k["ndc_cw"], k["ndc_ch"]
    t = -(F32(1) + pose[2]) / nds[:, 2]
    on = pose[None, :] + t[:, None] * nds
    q0, q1 = on[:, 0] / on[:, 2], on[:, 1] / on[:, 2]
    dd = np.stack([cw * (nds[:, 0] / nds[:, 2] - q0), ch * (nds[:, 1] / nds[:, 2] - q1), F32(-2) / on[:, 2]], -1)
    return ray_o, nds, dd
