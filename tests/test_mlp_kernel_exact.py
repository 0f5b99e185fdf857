"""Both MLP kernels against the bf16-faithful emulation (oracle/mlp_emulation.py):

  * bit for bit on exactly-summing networks, at row counts that leave every CTA of the persistent grid 0, 1 or 3+ tiles
    (the ring stage / phase carried across tiles, re-loaded tile inputs, the view-block swap on later tiles);
  * row by row on the shipped, shaped and random networks fed a whole 800x800 frame, with bounds set from H100
    measurements;
  * a rendered frame equals the same frame composed from the stage entry points, bit for bit."""
import pytest
import torch

from conftest import case_weights, load_golden, load_pavillon_weights
from oracle import adanerf_oracle as orc
from oracle import mlp_emulation as me

pytestmark = pytest.mark.gpu



def _row_counts():
    """Around one tile, around one tile per SM of the persistent grid (the device's SM count, as the library sizes the
    grid), and every CTA running 3+ tiles with a ragged last one."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return [1, 127, 128, 129, sms * 128 - 1, sms * 128 + 1, 3 * sms * 128 + 77]


def _renderer(scene, sd0=None, sd1=None):
    from adanerf_b200 import Renderer
    return Renderer(scene, device=0, sampling_net=sd0, shading_net=sd1)


@pytest.fixture(scope="module")
def bare():
    r = _renderer(orc.SCENE_BARBERSHOP)
    yield r
    r.close()


@pytest.fixture
def make_renderer():
    """Renderers that are closed (their frame-sized buffers freed) when the test ends, whether or not it passed."""
    made = []

    def make(scene, sd0=None, sd1=None):
        made.append(_renderer(scene, sd0, sd1))
        return made[-1]
    yield make
    for r in made:
        r.close()


def _first_difference(out, ref):
    bad = torch.nonzero((out != ref).any(1)).flatten()
    i = int(bad[0])
    return f"{bad.numel()} rows differ, first row {i} (tile {i // 128}): {out[i, :4].tolist()} != {ref[i, :4].tolist()}"


# ------------------------------------------------------------------------------------------------ bit-exact wiring
@pytest.mark.parametrize("terms", [3, 1])
@pytest.mark.parametrize("shape", me.EXACT_SAMPLING_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_mlp0_bit_exact_on_exact_nets(bare, shape, terms):
    n_in, depth, n_out = shape
    rows = _row_counts()
    sd, x = me.exact_sampling_net(n_in, depth, n_out, terms, rows=rows[-1], device="cuda")
    bare.set_option("mlp0_terms", terms)
    try:
        bare.set_weights(0, sd)
        ref = me.mlp0_emulate(x, sd, terms=terms)
        for n in rows:
            out = bare.mlp0(x[:n])
            assert torch.equal(out, ref[:n]), f"{n} rows: " + _first_difference(out, ref[:n])
    finally:
        bare.set_option("mlp0_terms", 3)


def test_mlp1_bit_exact_on_exact_net(bare):
    rows = _row_counts()
    sd, x = me.exact_shading_net(rows=rows[-1], device="cuda")
    bare.set_weights(1, sd)
    ref = me.mlp1_emulate(x, sd)
    for n in rows:
        out = bare.mlp1(x[:n])
        assert torch.equal(out, ref[:n]), f"{n} rows: " + _first_difference(out, ref[:n])


# ------------------------------------------------------------------------------------ full-frame numerics, every row
def _frame_case(kind):
    if kind == "pav":
        sd0, sd1 = load_pavillon_weights()
        return orc.SCENE_PAVILLON, sd0, sd1
    if kind == "barber":
        from test_shipped_models import load_barbershop_weights
        sd0, sd1 = load_barbershop_weights()
        return orc.SCENE_BARBERSHOP, sd0, sd1
    sd0, sd1 = orc.make_weights(kind, seed=0)
    return orc.SCENE_BARBERSHOP, sd0, sd1


# kind: (split net max rel, shading max rel, shading mean rel, shading fraction of rows above a bf16 flip), each 2x to
# 3.2x the value measured on an H100 80GB HBM3 (see the docstring below), rounded up.
FRAME_BOUNDS = {
    "pav": (4e-5, 1.5e-2, 1e-5, 1e-3),
    "barber": (4e-5, 2.5e-2, 9e-6, 9e-4),
    "shaped": (3e-5, 2.5e-2, 5e-5, 2e-2),
    "rand": (3.5e-5, 2.5e-2, 5e-5, 2e-2),
}


@pytest.mark.parametrize("kind", ["pav", "barber", "shaped", "rand"])
def test_mlp_kernels_full_frame_against_emulation(kind, make_renderer):
    """Stage 0 / stage 3 features of a whole 800x800 frame at thr 0.2, K = 8 (640 k sampling rows, ~5 M shading rows)
    through both kernels, every row compared with the float64 emulation on the device.  The kernels accumulate in fp32
    in the tensor cores' order, so they differ from the emulation by fp32 accumulation error only:
      split net:   max |raw0 - emu| / max |emu|;
      shading net: per output column, max and mean |raw1 - emu| / max |emu|, and the fraction of rows with an error
                   above 2^-9 of the column's scale (the size of one activation whose bf16 rounding flipped).
    Measured on an H100 80GB HBM3 at a 700 W power limit (shading rows: pav 5.12 M, barber 5.12 M, shaped 4.50 M,
    rand 5.12 M):
      kind    split max rel  shading max rel  shading mean rel  rows above a flip
      pav     1.87e-5        7.39e-3          3.47e-6           3.18e-4
      barber  1.79e-5        1.17e-2          3.11e-6           2.95e-4
      shaped  1.29e-5        1.15e-2          2.20e-5           8.18e-3
      rand    1.53e-5        1.13e-2          2.17e-5           7.98e-3
    The max statistics are set by the fp32 accumulation order and by the few rows where it flips a bf16 rounding of a
    hidden activation; the mean and the flip fraction are what a systematic error (a rounding mode, a dropped product,
    a dropped input band) moves.  The two trained nets (pav, barber: the reference's shipped Pavillon and Barbershop) agree
    on those two; barber's shading max is at the level of the synthetic nets'."""
    scene, sd0, sd1 = _frame_case(kind)
    r = make_renderer(scene, sd0, sd1)
    pose, rot = torch.tensor(scene["view_cell_center"]), torch.eye(3)
    dirs = r.generate_ray_directions(800, 800)
    x0, ro, rd = r.stage0(pose, rot, dirs)
    raw0 = r.mlp0(x0)
    emu0 = me.mlp0_emulate(x0, sd0, terms=3, chunk_rows=1 << 17)
    rel0 = float((raw0.double() - emu0.double()).abs().max() / emu0.abs().max())
    s2 = r.stage2(raw0, 0.2, 8)
    x1 = r.stage3(ro, rd, s2["ray"], s2["z"])
    del x0, emu0
    raw1 = r.mlp1(x1)
    emu1 = me.mlp1_emulate(x1, sd1, chunk_rows=1 << 18)
    scale = emu1.double().abs().amax(0)
    err = (raw1.double() - emu1.double()).abs() / scale
    max_rel = float(err.max())
    mean_rel = float(err.mean())
    frac = float((err > 2.0 ** -9).any(1).double().mean())
    print(f"{kind}: sampling rows {raw0.shape[0]}, shading rows {raw1.shape[0]}: split max rel {rel0:.3e}; "
          f"shading max rel {max_rel:.3e} per column {err.amax(0).tolist()}, mean rel {mean_rel:.3e}, "
          f"rows above a bf16 flip {frac:.3e}")
    b0, b1, b2, b3 = FRAME_BOUNDS[kind]
    assert rel0 < b0 and max_rel < b1 and mean_rel < b2 and frac < b3


# ------------------------------------------------------------------------------------------- composition invariant
def _compose(r, pose, rot, dirs, thr, K):
    """The frame from the stage entry points: stage 0 -> mlp0 -> stage 2 -> stage 3 -> mlp1 -> stage 5."""
    x0, ro, rd = r.stage0(pose, rot, dirs)
    raw0 = r.mlp0(x0)
    s2 = r.stage2(raw0, thr, K)
    x1 = r.stage3(ro, rd, s2["ray"], s2["z"])
    raw1 = r.mlp1(x1)
    out = r.stage5(raw1, s2["zp"], s2["z"], s2["offset"], s2["count"], K)
    return dict(rgb=out["rgb"], n_samples=s2["count"], raw0=raw0)


def _render_case(kind):
    """Scene, weights, pose, rotation and (thr, K) settings of a render-equals-stages case.  "terms1": the shaped nets
    with a plain bf16 sampling net (mlp0_terms = 1); "ndc": the golden NDC case (30-feature sampling net, ndc_rays in
    stage 3)."""
    if kind == "ndc":
        g = load_golden("ndc_k16_t0.15")
        m = g["meta"]
        sd0, sd1 = case_weights("ndc_k16_t0.15")
        return m["scene_params"], sd0, sd1, torch.from_numpy(g["pose"]), torch.from_numpy(g["rot"]), ((m["thr"], m["K"]),)
    scene, sd0, sd1 = _frame_case("shaped" if kind == "terms1" else kind)
    return scene, sd0, sd1, torch.tensor(scene["view_cell_center"]), orc.rotation_yaw(30.0), ((0.2, 8), (0.15, 16))


@pytest.mark.parametrize("kind", ["shaped", "pav", "terms1", "ndc"])
def test_render_equals_its_stages(kind, make_renderer):
    """render_rays / render_camera (device row counts, all-SM grids, stage 0 writing the sampling tiles, stage 3 writing
    the shading tiles or the fused encoder, chunking) == the stage entry points composed by hand, bit for bit."""
    scene, sd0, sd1, pose, rot, settings = _render_case(kind)
    r = make_renderer(scene, sd0, sd1)
    if kind == "terms1":
        r.set_option("mlp0_terms", 1)
    W = H = 800
    dirs = r.generate_ray_directions(W, H)
    for thr, K in settings:
        ref = _compose(r, pose, rot, dirs, thr, K)
        for fuse in (0, 1):
            r.set_option("fuse_encoder", fuse)
            out = r.render_rays(pose, rot, dirs, thr, K, want_oracle_weights=True)
            tag = f"{kind} thr {thr} K {K} fuse_encoder {fuse}"
            assert torch.equal(out["oracle_weights"], ref["raw0"]), tag
            assert torch.equal(out["n_samples"], ref["n_samples"]), tag
            assert torch.equal(out["rgb"], ref["rgb"]), tag
            cam = r.render_camera(pose, rot, W, H, thr, K, want_nsamples=True)
            assert torch.equal(cam["rgb"], ref["rgb"]) and torch.equal(cam["n_samples"], ref["n_samples"]), tag
        r.set_option("fuse_encoder", 0)
    r.set_option("chunk_rays", 50_000)
    out = r.render_rays(pose, rot, dirs, 0.2, 8, want_oracle_weights=True)
    r.set_option("chunk_rays", 0)
    ref = _compose(r, pose, rot, dirs, 0.2, 8)
    assert torch.equal(out["oracle_weights"], ref["raw0"]) and torch.equal(out["rgb"], ref["rgb"])
    # dense K = 128 on a few rows: z from the render's own z_vals
    d = dirs[:3 * W]
    x0, ro, rd = r.stage0(pose, rot, d)
    raw0 = r.mlp0(x0)
    n = d.shape[0]
    cnt = torch.full((n,), 128, dtype=torch.int32, device=d.device)
    off = (torch.arange(n, dtype=torch.int32, device=d.device) * 128)
    ray = torch.arange(n, dtype=torch.int32, device=d.device).repeat_interleave(128)
    for fuse in (0, 1):
        r.set_option("fuse_encoder", fuse)
        out = r.render_rays(pose, rot, d, 0.0, 128, want_oracle_weights=True, want_aux=("z_vals",))
        z = out["z_vals"].reshape(-1)
        raw1 = r.mlp1(r.stage3(ro, rd, ray, z))
        ref = r.stage5(raw1, raw0.reshape(-1), z, off, cnt, 128)
        assert torch.equal(out["oracle_weights"], raw0), f"dense fuse_encoder {fuse}"
        assert torch.equal(out["rgb"], ref["rgb"]), f"dense fuse_encoder {fuse}"
    r.set_option("fuse_encoder", 0)
