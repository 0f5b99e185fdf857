"""The sampling network's view (the C++ viewer's render-oracle mode) without a GPU: the numpy emulation against an
independent restatement of the reference kernel's order, the C++ host surface the viewer's NeuralRenderer compiles
against, the exported symbol and the headless viewer's --oracle flag."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from conftest import ROOT
from oracle import sampling_view as sv

NAN_POS = np.uint32(0x7FC00000).view(np.float32)
NAN_NEG = np.uint32(0xFFC00000).view(np.float32)


def restated(raw0):
    """cub::BlockRadixSort(...).SortDescending restated: a stable ascending sort of the complemented twiddled keys (the
    CUB of CUDA 12.x ranks -0 as +0), then the first three cells drawn as the viewer draws them."""
    b = np.asarray(raw0, np.float32).reshape(-1, 128).view(np.uint32).astype(np.uint64)
    b = np.where(b == 0x80000000, 0, b)                                     # -0 -> +0
    tw = np.where(b >= 0x80000000, 0xFFFFFFFF - b, b + 0x80000000)          # twiddle: order of the floats, NaNs outermost
    order = np.argsort(0xFFFFFFFF - tw, axis=1, kind="stable")[:, :3]
    rgb = (np.float32(0.5) + order.astype(np.float32)) / np.float32(128)
    px = np.concatenate([(np.clip(rgb, 0, 1) * np.float32(255)).astype(np.uint8), np.full((len(rgb), 1), 255, np.uint8)], 1)
    return order, rgb, px


def crafted_rows(seed=0):
    """Rows with ties of 2-128 cells, +-0 mixes, +-inf, NaNs of both signs, subnormals, all-equal rows and random rows."""
    rng = np.random.default_rng(seed)
    rows = [rng.standard_normal(128).astype(np.float32) for _ in range(64)]
    for n_tie in (2, 3, 4, 7, 8, 9, 16, 33, 64, 127, 128):
        r = rng.standard_normal(128).astype(np.float32) - 5
        r[rng.choice(128, n_tie, replace=False)] = np.float32(rng.choice([0.25, -1.5, 3.0]))
        rows.append(r)
    for fill in (0.0, -0.0, 1.0, -np.inf, np.inf, NAN_POS, NAN_NEG, np.float32(1e-45)):
        rows.append(np.full(128, fill, np.float32))
    zeros = np.where(rng.random(128) < 0.5, np.float32(0.0), np.float32(-0.0)).astype(np.float32)
    rows.append(zeros)
    z2 = zeros.copy()
    z2[rng.choice(128, 5, replace=False)] = -1e-40                                # negative subnormals under the zeros
    rows.append(z2)
    specials = np.array([np.inf, -np.inf, NAN_POS, NAN_NEG, 0.0, -0.0, 1e-45, -1e-45, 1e-38, -1e-38], np.float32)
    for _ in range(24):
        rows.append(rng.choice(specials, 128).astype(np.float32))
        r = rng.standard_normal(128).astype(np.float32)
        r[rng.choice(128, 6, replace=False)] = rng.choice(specials, 6)
        rows.append(r)
    payload = np.uint32(0x7F800001 + rng.integers(0, 1 << 22, 128)).view(np.float32)   # NaNs of many payloads
    rows.append(payload)
    rows.append(-payload)
    q = np.round(rng.standard_normal(128) * 2).astype(np.float32)                 # a few values, many ties each
    rows.append(q)
    return np.stack(rows).astype(np.float32)


def test_emulation_equals_the_restated_radix_order():
    raw0 = np.concatenate([crafted_rows(0), np.random.default_rng(1).standard_normal((4096, 128)).astype(np.float32)])
    order, rgb, px = restated(raw0)
    assert np.array_equal(sv.top3(raw0), order)
    got_rgb, got_px = sv.sampling_view(raw0)
    assert np.array_equal(got_rgb.view(np.uint32), rgb.view(np.uint32))
    assert np.array_equal(got_px, px)


def test_emulation_rules_on_special_values():
    row = np.full(128, -1.0, np.float32)
    row[[5, 9, 40]] = [NAN_NEG, -np.inf, np.inf]
    row[[70, 71]] = NAN_POS
    assert sv.top3(row).tolist() == [[70, 71, 40]]                   # +NaN above +inf, ties lower cell first
    row = np.full(128, -np.inf, np.float32)
    row[[3, 100]] = NAN_NEG
    row[7] = -0.0
    row[2] = 0.0
    assert sv.top3(row).tolist() == [[2, 7, 0]]                      # -0 ties +0 (lower cell first), -NaN below -inf
    assert sv.top3(np.full(128, 0.5, np.float32)).tolist() == [[0, 1, 2]]
    rgb, px = sv.sampling_view(np.arange(128, dtype=np.float32)[::-1].copy())
    assert rgb.tolist() == [[0.5 / 128, 1.5 / 128, 2.5 / 128]]
    assert px.tolist() == [[int(np.float32(0.5 / 128) * np.float32(255)), int(np.float32(1.5 / 128) * np.float32(255)),
                            int(np.float32(2.5 / 128) * np.float32(255)), 255]]


def test_symbol_is_exported():
    import __graft_entry__ as g
    g.build()
    lib = ctypes.CDLL(g.LIB)
    assert hasattr(lib, "adn_sampling_view")
    from adanerf_b200._lib import SYMBOLS
    assert "adn_sampling_view" in SYMBOLS


NEURAL_RENDERER_TU = r"""
// The calls the viewer's NeuralRenderer makes on its ImageGenerator (include/neuralrenderer.h:65, neuralrenderer.cpp),
// against adn_host::ImageGenerator.
#include <vector>
#include "image_generator.h"
class FeatureSet {};
class Encoding {};
struct NeuralRendererLike {
  adn_host::ImageGenerator img_gen;
  adn_host::Config config;
  adn_host::Camera camera;
  std::vector<FeatureSet*> feature_sets;
  std::vector<Encoding> encodings;
  bool init() { return img_gen.load(config); }
  bool render(unsigned long long surf, int batch_size, int num_samples) {
    return img_gen.inference(camera, surf, batch_size, num_samples, feature_sets, encodings);
  }
  void switchRenderOracle() { img_gen.switchRenderOracle(); }
  bool oracleOn() const { return img_gen.renderOracle(); }
};
int main() {
  NeuralRendererLike r;
  r.switchRenderOracle();
  return r.oracleOn() ? 0 : 1;
}
"""


def test_neural_renderer_calls_compile(tmp_path):
    src = tmp_path / "neural_renderer_like.cpp"
    src.write_text(NEURAL_RENDERER_TU)
    inc = os.path.join(ROOT, "adanerf_b200", "csrc", "host")
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-I" + inc, str(src)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


@pytest.fixture(scope="module")
def viewer():
    import __graft_entry__ as g
    g.build()
    return g.VIEWER


def test_headless_viewer_accepts_oracle_and_fails_loudly_without_gpu(viewer, tmp_path):
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from adanerf_b200 import onnx_weights as ow
    from oracle import adanerf_oracle as orc
    sd0, sd1 = orc.make_weights("shaped", seed=0)
    d = str(tmp_path / "export")
    ow.write_export_dir(d, orc.SCENE_BARBERSHOP, sd0, sd1, 0.2, 8)
    r = subprocess.run([viewer, d, "--oracle", "--surface", "-f", "1"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 1 and "usage" not in r.stderr
    assert "no usable sm_90 device" in r.stderr
    r = subprocess.run([viewer, d, "--oracle-typo"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 2 and "[--oracle]" in r.stderr
