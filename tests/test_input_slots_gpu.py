"""The shading kernel's input slots: its producer warps fill the next tile's inputs while the consumers run the current
one, by encoding the samples (option fuse_encoder = 1, the default for non-NDC scenes) or by one bulk copy of the packed
tile stage 3 wrote (fuse_encoder = 0).  Both render the frame the stage entry points compose by hand, bit for bit:

  * the default, with no option set, against fuse_encoder 0 and the stage entries, adaptive and dense K = 128;
  * a three-block encoding (posEncArgs 20-10: [P0 | P1 | V], whose two slots take two weight-ring stages' room);
  * sample totals that leave the persistent grid's CTAs 0, 1, 2 and 3 tiles (dense totals are exact: one tile per ray),
    and adaptive totals that are not multiples of 128;
  * a call of several chunks."""
import pytest
import torch

from oracle import adanerf_oracle as orc
from test_encodings import CASES, case_scene, case_weights
from test_mlp_kernel_exact import _compose

pytestmark = pytest.mark.gpu

W = H = 800


@pytest.fixture
def make_renderer():
    made = []

    def make(scene, sd0=None, sd1=None):
        from adanerf_b200 import Renderer
        made.append(Renderer(scene, device=0, sampling_net=sd0, shading_net=sd1))
        return made[-1]
    yield make
    for r in made:
        r.close()


def _case(kind, make_renderer):
    if kind == "p20-10":
        name, fields, shape = CASES[0]
        assert name == "s10-4_p20-10"
        scene = case_scene(fields)
        sd0, sd1 = case_weights(scene, shape)
    else:
        scene = orc.SCENE_BARBERSHOP
        sd0, sd1 = orc.make_weights("shaped", seed=0)
    r = make_renderer(scene, sd0, sd1)
    return r, torch.tensor(scene["view_cell_center"], dtype=torch.float32), orc.rotation_yaw(25.0)


def _renders(r, pose, rot, dirs, thr, K, **kw):
    """The default render, then the tile path's (fuse_encoder 0); the default restored."""
    out = r.render_rays(pose, rot, dirs, thr, K, **kw)
    r.set_option("fuse_encoder", 0)
    try:
        tiles = r.render_rays(pose, rot, dirs, thr, K, **kw)
    finally:
        r.set_option("fuse_encoder", 1)
    return out, tiles


def _dense_stages(r, pose, rot, d, z):
    """A dense K = 128 frame from the stage entry points, z = the render's z_vals."""
    x0, ro, rd = r.stage0(pose, rot, d)
    raw0 = r.mlp0(x0)
    n = d.shape[0]
    ray = torch.arange(n, dtype=torch.int32, device=d.device).repeat_interleave(128)
    cnt = torch.full((n,), 128, dtype=torch.int32, device=d.device)
    off = torch.arange(n, dtype=torch.int32, device=d.device) * 128
    raw1 = r.mlp1(r.stage3(ro, rd, ray, z))
    return r.stage5(raw1, raw0.reshape(-1), z, off, cnt, 128)["rgb"]


@pytest.mark.parametrize("kind", ["p10-4", "p20-10"])
def test_default_render_equals_tile_path_and_stages(kind, make_renderer):
    r, pose, rot = _case(kind, make_renderer)
    dirs = r.generate_ray_directions(W, H)
    for thr, K in ((0.2, 8), (0.15, 16)):
        ref = _compose(r, pose, rot, dirs, thr, K)
        out, tiles = _renders(r, pose, rot, dirs, thr, K)
        tag = f"{kind} thr {thr} K {K}"
        assert torch.equal(out["n_samples"], ref["n_samples"]) and torch.equal(tiles["n_samples"], ref["n_samples"]), tag
        assert torch.equal(out["rgb"], ref["rgb"]), tag + ": default"
        assert torch.equal(tiles["rgb"], ref["rgb"]), tag + ": fuse_encoder 0"
        cam = r.render_camera(pose, rot, W, H, thr, K)
        assert torch.equal(cam["rgb"], ref["rgb"]), tag + ": render_camera"


@pytest.mark.parametrize("kind", ["p10-4", "p20-10"])
def test_tiles_per_cta_from_zero_to_three(kind, make_renderer):
    """Dense K = 128 renders of n rays run exactly n tiles on the all-SM grid: n = sms / 2 leaves CTAs with 0 and 1 tile,
    sms + 1 with 1 and 2, 2 sms + 1 with 2 and 3, 3 sms with 3 each.  Then adaptive renders with ragged sample totals."""
    r, pose, rot = _case(kind, make_renderer)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    dirs = r.generate_ray_directions(W, H)
    for n in (sms // 2, sms + 1, 2 * sms + 1, 3 * sms):
        d = dirs[::(W * H) // n][:n].contiguous()
        out, tiles = _renders(r, pose, rot, d, 0.0, 128, want_aux=("z_vals",))
        ref = _dense_stages(r, pose, rot, d, out["z_vals"].reshape(-1))
        assert torch.equal(out["z_vals"], tiles["z_vals"]), f"dense {n} rays"
        assert torch.equal(out["rgb"], ref), f"dense {n} rays: default"
        assert torch.equal(tiles["rgb"], ref), f"dense {n} rays: fuse_encoder 0"
    ragged = 0
    for n in (300, 2500, 6000, 9000):
        d = dirs[::(W * H) // n][:n].contiguous()
        ref = _compose(r, pose, rot, d, 0.2, 8)
        out, tiles = _renders(r, pose, rot, d, 0.2, 8)
        m = int(ref["n_samples"].sum())
        ragged += m % 128 != 0
        print(f"{kind}: {n} rays, {m} samples, {(m + 127) // 128} tiles over {sms} CTAs")
        assert torch.equal(out["rgb"], ref["rgb"]) and torch.equal(tiles["rgb"], ref["rgb"]), f"{n} rays"
    assert ragged > 0


def test_multi_chunk_call(make_renderer):
    r, pose, rot = _case("p10-4", make_renderer)
    dirs = r.generate_ray_directions(W, H)
    whole = r.render_rays(pose, rot, dirs, 0.2, 8)
    r.set_option("chunk_rays", 50_000)
    try:
        out, tiles = _renders(r, pose, rot, dirs, 0.2, 8)
        cam = r.render_camera(pose, rot, W, H, 0.2, 8)
    finally:
        r.set_option("chunk_rays", 0)
    ref = _compose(r, pose, rot, dirs, 0.2, 8)
    for what, rgb in (("one chunk", whole["rgb"]), ("chunks", out["rgb"]), ("chunks, fuse_encoder 0", tiles["rgb"]),
                      ("chunks, render_camera", cam["rgb"])):
        assert torch.equal(rgb, ref["rgb"]), what
