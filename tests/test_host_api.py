"""Host-side behaviour of the public entry points (GPU): render() always uses the current parameters, explicit host
buffer registration, several contexts in one process."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import adanerf_oracle as orc

pytestmark = pytest.mark.gpu


def _nets(seed):
    """nn.Modules with the reference's parameter names (src/models.py:71-76, 226-244)."""
    sd0, sd1 = orc.make_weights("shaped", seed=seed)

    class Net(torch.nn.Module):
        def __init__(self, sd):
            super().__init__()
            for k, v in sd.items():
                self.register_parameter(k.replace(".", "__"), torch.nn.Parameter(v.clone(), requires_grad=False))
            self._names = list(sd)

        def state_dict(self, *a, **kw):
            return {k: getattr(self, k.replace(".", "__")) for k in self._names}

    return Net(sd0), Net(sd1)


def _rays(n=2048):
    scene = orc.SCENE_BARBERSHOP
    dirs = torch.from_numpy(orc.generate_ray_directions(800, 800, scene["fov"]).reshape(-1, 3)).float()[::311][:n]
    return dict(pose=torch.tensor(scene["view_cell_center"]), rot=orc.rotation_yaw(30.0), dirs=dirs.cuda())


def test_render_uses_the_current_parameters():
    """The reference's inference() always runs the live modules (src/train_data.py:278-299); render() caches the packed
    device copy but must notice in-place updates and freshly loaded networks (ADVICE r1: the cache was keyed on id())."""
    from adanerf_b200 import render, Renderer
    scene = orc.SCENE_BARBERSHOP
    rays = _rays()
    n0, n1 = _nets(0)
    a, _ = render(rays, n0, n1, 0.2, K=8, scene=scene)
    again, _ = render(rays, n0, n1, 0.2, K=8, scene=scene)
    assert torch.equal(a, again)
    with torch.no_grad():                                   # eval during training: optimizer steps write in place
        n1.state_dict()["rgb_linear.bias"].add_(0.25)
    b, _ = render(rays, n0, n1, 0.2, K=8, scene=scene)
    fresh = Renderer(scene, device=0, sampling_net=n0, shading_net=n1)
    want = fresh.render_rays(rays["pose"], rays["rot"], rays["dirs"], 0.2, 8)["rgb"]
    fresh.close()
    assert not torch.equal(a, b) and torch.equal(b, want)
    # a loop over checkpoints: new module objects every time, the old ones garbage collected (ids may be recycled)
    for seed in (1, 2, 3):
        m0, m1 = _nets(seed)
        got, _ = render(rays, m0, m1, 0.2, K=8, scene=scene)
        fresh = Renderer(scene, device=0, sampling_net=m0, shading_net=m1)
        want = fresh.render_rays(rays["pose"], rays["rot"], rays["dirs"], 0.2, 8)["rgb"]
        fresh.close()
        assert torch.equal(got, want), seed
        del m0, m1


def test_host_buffers_registered_explicitly_or_staged():
    """render_rays_host / render_camera_host: identical results whether the arrays are registered (DMA in place), plain
    (staged), or temporaries created by a dtype conversion that die right after the call (ADVICE r1: implicit
    cudaHostRegister on such temporaries left stale registrations behind)."""
    from adanerf_b200 import Renderer
    scene = orc.SCENE_BARBERSHOP
    sd0, sd1 = orc.make_weights("shaped", seed=0)
    r = Renderer(scene, device=0, sampling_net=sd0, shading_net=sd1)
    rays = _rays(4096)
    dirs = np.ascontiguousarray(rays["dirs"].cpu().numpy())
    ref = r.render_rays(rays["pose"], rays["rot"], rays["dirs"], 0.2, 8)
    out = np.empty((dirs.shape[0], 3), np.float32)
    r.register_host_buffer(dirs)
    r.register_host_buffer(out)
    for _ in range(3):
        got = r.render_rays_host(rays["pose"], rays["rot"], dirs, 0.2, 8, out=out)
        assert got["rgb"] is out
        np.testing.assert_array_equal(out, ref["rgb"].cpu().numpy())
        np.testing.assert_array_equal(got["n_samples"], ref["n_samples"].cpu().numpy())
    with pytest.raises(Exception):
        r.register_host_buffer(out)                         # twice
    r.unregister_host_buffer(out)
    r.unregister_host_buffer(dirs)
    with pytest.raises(Exception):
        r.unregister_host_buffer(dirs)                      # not registered any more
    for _ in range(4):                                      # float64 input: a fresh float32 temporary inside every call
        got = r.render_rays_host(rays["pose"], rays["rot"], dirs.astype(np.float64), 0.2, 8)
        np.testing.assert_array_equal(got["rgb"], ref["rgb"].cpu().numpy())
        junk = [np.empty(dirs.shape, np.float32) for _ in range(3)]   # churn the allocator between calls
        del junk
    # render_camera_host == render_camera, into plain (staged) arrays and into registered ones (DMA in place)
    W, H, row0, rows = 800, 800, 300, 64
    cam = r.render_camera(rays["pose"], rays["rot"], W, H, 0.2, 8, row0=row0, rows=rows, want_nsamples=True)
    want_rgb, want_ns = cam["rgb"].cpu().numpy(), cam["n_samples"].cpu().numpy()
    plain = r.render_camera_host(rays["pose"], rays["rot"], W, H, 0.2, 8, row0=row0, rows=rows, want_nsamples=True)
    np.testing.assert_array_equal(plain["rgb"], want_rgb)
    np.testing.assert_array_equal(plain["n_samples"], want_ns)
    rgb, ns = np.empty((rows * W, 3), np.float32), np.empty((rows * W,), np.int32)
    r.register_host_buffer(rgb)
    r.register_host_buffer(ns)
    p, q = (np.ascontiguousarray(np.asarray(x, np.float32).reshape(-1)) for x in (rays["pose"], rays["rot"]))
    assert r.lib.adn_render_camera_host(r.handle, p.ctypes.data_as(ctypes.POINTER(ctypes.c_float)),
                                        q.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), W, H, row0, rows, 0.2, 8,
                                        rgb.ctypes.data, ns.ctypes.data) == 0
    np.testing.assert_array_equal(rgb, want_rgb)
    np.testing.assert_array_equal(ns, want_ns)
    r.close()


def test_sampling_net_output_width_is_checked():
    from adanerf_b200 import Renderer
    r = Renderer(orc.SCENE_BARBERSHOP, device=0)
    g = torch.Generator().manual_seed(3)
    r.set_option("mlp0_terms", 1)
    r.set_weights(0, {"layers.0.weight": torch.randn(256, 90, generator=g), "layers.0.bias": torch.zeros(256)})
    assert r.net_dims(0) == (90, 256)
    x = torch.randn(100, 90, generator=g).cuda()
    assert r.mlp0(x).shape == (100, 256)                    # sized from the network, not from a caller's guess
    with pytest.raises(ValueError):
        r.mlp0(x, n_out=128)
    r.close()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_contexts_on_two_devices_in_one_process():
    """cudaFuncAttributeMaxDynamicSharedMemorySize is a per-device attribute (ADVICE r1: a process-wide flag skipped it
    on the second device and its MLP launches failed)."""
    from adanerf_b200 import Renderer
    scene = orc.SCENE_BARBERSHOP
    sd0, sd1 = orc.make_weights("shaped", seed=0)
    rays = _rays(4096)
    outs = []
    for dev in (0, 1):
        r = Renderer(scene, device=dev, sampling_net=sd0, shading_net=sd1)
        o = r.render_rays(rays["pose"], rays["rot"], rays["dirs"].to(f"cuda:{dev}"), 0.2, 8)
        outs.append((o["rgb"].cpu(), o["n_samples"].cpu()))
        r.close()
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
