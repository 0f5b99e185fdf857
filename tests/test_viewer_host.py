"""C++ host program (adanerf_b200/csrc/host): builds with plain g++ against the C ABI; fails loudly without a
GPU; on an H100 renders an export directory end to end."""
import os
import re
import subprocess

import pytest
import torch

from adanerf_b200 import onnx_weights as ow
from oracle import adanerf_oracle as orc


@pytest.fixture(scope="module")
def viewer():
    import __graft_entry__ as g
    g.build()
    assert os.path.exists(g.VIEWER)
    return g.VIEWER


def _export(tmp_path):
    sd0, sd1 = orc.make_weights("shaped", seed=0)
    d = tmp_path / "export"
    ow.write_export_dir(str(d), orc.SCENE_BARBERSHOP, sd0, sd1, 0.2, 8)
    return str(d)


def test_viewer_fails_loudly_without_gpu(viewer, tmp_path):
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    r = subprocess.run([viewer, _export(tmp_path), "-f", "1"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 1
    assert "K = 8" in r.stdout and "no usable sm_90 device" in r.stderr


def test_viewer_rejects_missing_dir(viewer, tmp_path):
    r = subprocess.run([viewer, str(tmp_path / "nope")], capture_output=True, text=True, timeout=120)
    assert r.returncode == 1 and "couldn't read export directory" in r.stderr


@pytest.mark.gpu
def test_viewer_renders_export_dir(viewer, tmp_path):
    d = _export(tmp_path)
    r = subprocess.run([viewer, d, "-s", "400", "300", "-f", "5", "-w"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    m = re.search(r"5 frames 400x300: ([0-9.]+) ms/frame .*\(([0-9.]+) per ray", r.stdout)
    assert m, r.stdout
    assert 1.0 <= float(m.group(2)) <= 8.0
    ppm = open(os.path.join(d, "adn_frame.ppm"), "rb").read()
    assert ppm.startswith(b"P6\n400 300\n255\n") and len(ppm) == len(b"P6\n400 300\n255\n") + 400 * 300 * 3


@pytest.mark.gpu
def test_viewer_frame_through_a_surface_object(viewer, tmp_path):
    """ImageGenerator::inference(camera, cudaSurfaceObject_t, batch, K, feature_sets, encodings) -- the reference's
    parameter list (adanerf_real_time_viewer/include/imagegenerator.h:61-62) -- writes the uchar4 frame into a
    surface-bound cudaArray exactly like adaptive_cuda_kernels.cu:846-851; the program compares it with the fp32 frame."""
    d = _export(tmp_path)
    r = subprocess.run([viewer, d, "-s", "400", "300", "-f", "2", "--surface"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "surface frame 400x300: 0 mismatching bytes" in r.stdout, r.stdout


@pytest.mark.gpu
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_viewer_on_two_gpus_renders_the_same_frame(viewer, tmp_path):
    """C++ host, one process, two devices, NCCL gather (include/adanerf_b200_multi.h): same checksum as the bands rendered on
    one device."""
    d = _export(tmp_path)
    r2 = subprocess.run([viewer, d, "-s", "400", "301", "-f", "4", "-g", "2"], capture_output=True, text=True, timeout=300)
    assert r2.returncode == 0, r2.stdout + r2.stderr
    assert "on 2 GPUs" in r2.stdout and "checksum" in r2.stdout
