"""TEST INFRASTRUCTURE ONLY -- builds the reference viewer's CUDA kernels into oracle/_ref/libref_viewer_kernels.so.

The unmodified adanerf_real_time_viewer/src/cuda/base_cuda_kernels.cu of a local reference checkout
(ref_harness.REF_ROOT), compiled for sm_90a together with oracle/ref_viewer_shim.cu, which exports
ref_sampling_view(d_raw0, n_rays, width, d_px): the viewer's render-oracle picture (copyResultSamplingNetwork) read back
into linear uchar4 pixels.  The GPU tests compare our sampling_view_kernel with it byte for byte.

Without a reference checkout (e.g. on a machine that only runs the tests) build() does nothing: it never fails and never
deletes an artefact built earlier.  The artefact is keyed on the content of everything it is built from (sidecar
<artefact>.srchash), and it is written to a temporary file first and moved into place, so concurrent builds are safe."""
import hashlib
import os
import subprocess
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
OUT_DIR = os.path.join(HERE, "_ref")
LIB = os.path.join(OUT_DIR, "libref_viewer_kernels.so")
SHIM = os.path.join(HERE, "ref_viewer_shim.cu")
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-shared"]


def viewer_dir():
    from oracle.ref_harness import REF_ROOT
    return os.path.join(REF_ROOT, "adanerf_real_time_viewer")


def _inputs():
    """The files the artefact is built from: the viewer's kernel source and the headers it includes, and the shim."""
    v = viewer_dir()
    inc = os.path.join(v, "include", "cuda")
    return [os.path.join(v, "src", "cuda", "base_cuda_kernels.cu"), os.path.join(inc, "adanerf_cuda_kernels.cuh"),
            os.path.join(inc, "helper_math.h"), os.path.join(inc, "adanerf_cuda_helper.h"), SHIM]


def _digest(nvcc):
    h = hashlib.sha256()
    for f in _inputs():
        h.update(os.path.basename(f).encode())
        with open(f, "rb") as fh:
            h.update(fh.read())
    h.update(" ".join([nvcc] + NVCC_FLAGS).encode())
    return h.hexdigest()


def available():
    return all(os.path.isfile(f) for f in _inputs())


def build(nvcc="nvcc", force=False):
    """Compiles the artefact when a reference checkout exists and the artefact is missing or stale; else does nothing.
    Returns the artefact's path, or None when there is no reference checkout."""
    if not available():
        return None
    digest = _digest(nvcc)
    side = LIB + ".srchash"
    if not force and os.path.exists(LIB) and os.path.exists(side):
        with open(side) as fh:
            if fh.read().strip() == digest:
                return LIB
    os.makedirs(OUT_DIR, exist_ok=True)
    fd, tmp = tempfile.mkstemp(prefix=".libref_viewer_kernels.", suffix=".so", dir=OUT_DIR)
    os.close(fd)
    try:
        src = _inputs()[0]
        cmd = [nvcc] + NVCC_FLAGS + ["-I" + os.path.join(viewer_dir(), "include"), "-o", tmp, src, SHIM]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed building oracle/_ref/libref_viewer_kernels.so:\n" + r.stdout + r.stderr)
        os.replace(tmp, LIB)
        with open(side, "w") as fh:
            fh.write(digest + "\n")
    finally:
        if os.path.exists(tmp):
            os.unlink(tmp)
    return LIB
