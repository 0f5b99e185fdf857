"""The split-precision sampling MLP (mlp_kernel<2>) and its weight ring of [128 x 32] hi + lo stages, with each tile's
inputs bulk-copied while the previous tile finishes:

  * bit for bit against the bf16-faithful emulation on exactly-summing nets whose second input block holds 0-4 K steps
    (no stage, one stage, two stages) and whose stages per tile cover every residue modulo the 5-stage ring, at row
    counts that leave every CTA 0, 1 or 3+ tiles with a ragged last one;
  * one whole 800x800 stage 0 -> mlp0 frame computed twice on one renderer is byte-identical (an input tile read before
    its copy landed would differ between the two)."""
import pytest
import torch

from oracle import mlp_emulation as me
from test_mlp_kernel_exact import _render_case

pytestmark = pytest.mark.gpu


def _row_counts():
    """Around one tile, around one tile per SM of the persistent grid (the device's SM count, as the library sizes the
    grid), and every CTA running 3+ tiles with a ragged last one."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return [1, 127, 128, 129, sms * 128 - 1, sms * 128 + 1, 3 * sms * 128 + 77]


def _stages_per_tile(n_in, depth, n_out, width=256):
    """Ring stages one tile takes (layer_stages in csrc/mlp.cuh): per N half, ceil(K steps / 2) per K block."""
    def block_stages(valid):
        return (-(-valid // 16) + 1) // 2
    first = block_stages(min(64, n_in)) + block_stages(max(0, n_in - 64))
    total = 0
    for l in range(depth):
        halves = (n_out if l == depth - 1 else width) // 128
        total += halves * (first if l == 0 else (width // 64) * 2)
    return total


# (n_in, depth, n_out): second input block with 0 (30), 1 (65), 2 (90), 3 (100) and 4 (128) K steps; the 90-input nets'
# stages per tile are 3, 6, 14, 30, 38, 110 and 182, every residue modulo 5.
SHAPES = [(30, 2, 128), (65, 2, 128), (90, 2, 128), (100, 2, 128), (128, 2, 256),
          (90, 1, 128), (90, 1, 256), (90, 3, 128), (90, 3, 256), (90, 8, 128), (90, 12, 256)]


def test_shapes_cover_every_ring_residue():
    assert {_stages_per_tile(*s) % 5 for s in SHAPES} == set(range(5))


@pytest.fixture(scope="module")
def bare():
    from adanerf_b200 import Renderer
    from oracle import adanerf_oracle as orc
    r = Renderer(orc.SCENE_BARBERSHOP, device=0)
    yield r
    r.close()


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_split_mlp0_bit_exact(bare, shape):
    n_in, depth, n_out = shape
    rows = _row_counts()
    sd, x = me.exact_sampling_net(n_in, depth, n_out, 3, rows=rows[-1], device="cuda")
    bare.set_option("mlp0_terms", 3)
    bare.set_weights(0, sd)
    ref = me.mlp0_emulate(x, sd, terms=3)
    for n in rows:
        out = bare.mlp0(x[:n])
        bad = torch.nonzero((out != ref[:n]).any(1)).flatten()
        assert bad.numel() == 0, f"{n} rows: {bad.numel()} rows differ, first row {int(bad[0])} (tile {int(bad[0]) // 128})"


@pytest.mark.parametrize("kind", ["rand", "pav", "ndc"])
def test_split_mlp0_frame_twice_identical(kind):
    from adanerf_b200 import Renderer
    if kind == "rand":
        from test_mlp_kernel_exact import _frame_case
        scene, sd0, sd1 = _frame_case("rand")
        pose, rot = torch.tensor(scene["view_cell_center"]), torch.eye(3)
    else:
        scene, sd0, sd1, pose, rot, _ = _render_case(kind)
    r = Renderer(scene, device=0, sampling_net=sd0, shading_net=sd1)
    try:
        dirs = r.generate_ray_directions(800, 800)
        x0, _, _ = r.stage0(pose, rot, dirs)
        a = r.mlp0(x0).clone()
        b = r.mlp0(x0)
        torch.cuda.synchronize()
        assert torch.isfinite(a).all()
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), f"{kind}: {int((a != b).any(1).sum())} rows differ"
    finally:
        r.close()
