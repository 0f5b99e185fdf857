"""One process, several GPUs: adn_multi_* (include/adanerf_b200_multi.h) -- row bands, ncclCommInitAll, one gather per
frame.  The invariant of SURVEY.md 8e: the gathered frame equals the single-GPU frame bit for bit."""
import numpy as np
import pytest
import torch

from oracle import adanerf_oracle as orc

pytestmark = pytest.mark.gpu


def _single_frames(scene, sd0, sd1, poses, W, H):
    from adanerf_b200 import Renderer
    single = Renderer(scene, device=0, sampling_net=sd0, shading_net=sd1)
    want = [single.render_camera(p, r, W, H, 0.2, 8)["rgb"].cpu() for p, r in poses]
    single.close()
    return want


def _poses(scene, n):
    """n different views: each frame in flight has its own pose, so a slot mix-up in wait_frame shows."""
    c = torch.tensor(scene["view_cell_center"])
    return [(c + torch.tensor([0.05 * i, -0.03 * i, 0.01 * i]), orc.rotation_yaw(20.0 + 17.0 * i)) for i in range(n)]


def test_band_partition_on_one_device():
    """n_devices = 1 needs no communicator: the frame path (band buffer, copy into the frame, two frames in flight) alone.
    Two frames of different poses in flight come back in order; then a frame-size change with nothing in flight."""
    from adanerf_b200.multi import MultiRenderer
    scene = orc.SCENE_BARBERSHOP
    sd0, sd1 = orc.make_weights("shaped", seed=0)
    poses = _poses(scene, 3)
    want = _single_frames(scene, sd0, sd1, poses[:2], 320, 200)
    assert not torch.equal(want[0], want[1])
    m = MultiRenderer(scene, [0], sd0, sd1)
    assert m.band(200, 0) == (0, 200)
    m.render_camera(*poses[0], 320, 200, 0.2, 8)
    m.render_camera(*poses[1], 320, 200, 0.2, 8)
    with pytest.raises(Exception):
        m.render_camera(*poses[2], 320, 200, 0.2, 8)        # a third frame in flight
    a = m.wait_frame().cpu()
    host = np.empty((320 * 200, 3), np.float32)
    m.wait_frame(host_out=host)
    assert torch.equal(a, want[0]) and np.array_equal(host, want[1].numpy())
    small = _single_frames(scene, sd0, sd1, poses[2:], 256, 120)[0]
    m.render_camera(*poses[2], 256, 120, 0.2, 8)             # another frame size, nothing in flight
    assert torch.equal(m.wait_frame().cpu(), small)
    m.close()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
@pytest.mark.parametrize("H", [200, 203])
def test_gathered_frame_equals_single_gpu_frame(H):
    from adanerf_b200.multi import MultiRenderer
    scene = orc.SCENE_BARBERSHOP
    sd0, sd1 = orc.make_weights("shaped", seed=0)
    poses = _poses(scene, 5)
    G = min(torch.cuda.device_count(), 4)
    want = _single_frames(scene, sd0, sd1, poses[:4], 320, H)
    small = _single_frames(scene, sd0, sd1, poses[4:], 256, H - 81)[0]
    m = MultiRenderer(scene, list(range(G)), sd0, sd1)
    rows = [m.band(H, r) for r in range(G)]
    assert rows[0][0] == 0 and sum(n for _, n in rows) == H and all(rows[i][0] + rows[i][1] == rows[i + 1][0] for i in range(G - 1))
    m.render_camera(*poses[0], 320, H, 0.2, 8)
    for i in range(1, 4):                                   # pipelined: the next frame is enqueued before the previous is read
        m.render_camera(*poses[i], 320, H, 0.2, 8)
        got = m.wait_frame().cpu()
        assert torch.equal(got, want[i - 1]), f"frame {i - 1}"
    assert torch.equal(m.wait_frame().cpu(), want[3])
    m.render_camera(*poses[4], 256, H - 81, 0.2, 8)          # another frame size, nothing in flight
    assert torch.equal(m.wait_frame().cpu(), small)
    render_ms, gather_ms = m.last_times()
    assert len(render_ms) == G and all(t > 0 for t in render_ms)
    m.close()
