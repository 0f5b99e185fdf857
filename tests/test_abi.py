"""CPU-side checks: the C-ABI library builds for sm_90a, loads, and exports every symbol the header
declares; the product path fails loudly without a GPU (no CPU fallback)."""
import ctypes
import os
import re

import pytest

from conftest import ROOT


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    return ctypes.CDLL(g.LIB)


def test_library_exports_every_header_symbol(lib):
    hdr = open(os.path.join(ROOT, "include", "adanerf_b200.h")).read()
    declared = set(re.findall(r"\b(adn_[a-z0-9_]+)\s*\(", hdr))
    declared -= {"adn_ctx"}
    from adanerf_b200._lib import SYMBOLS
    assert declared == set(SYMBOLS), (declared ^ set(SYMBOLS))
    for s in declared:
        assert hasattr(lib, s), s


def test_multi_library_exports_every_header_symbol():
    """libadanerf_b200_multi.so (one process, G devices, NCCL gather): header == exports == ctypes shim."""
    import __graft_entry__ as g
    g.build()
    hdr = open(os.path.join(ROOT, "include", "adanerf_b200_multi.h")).read()
    declared = set(re.findall(r"\b(adn_multi_[a-z0-9_]+)\s*\(", hdr))
    from adanerf_b200.multi import SYMBOLS
    assert declared == set(SYMBOLS), (declared ^ set(SYMBOLS))
    mlib = ctypes.CDLL(g.MULTI_LIB)
    for s in declared:
        assert hasattr(mlib, s), s


def test_sass_is_hopper_native():
    """wgmma.mma_async -> HGMMA, bulk async copy -> UBLKCP."""
    import shutil
    import subprocess
    import __graft_entry__ as g
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", g.LIB], capture_output=True, text=True).stdout
    assert "sm_90a" in sass
    for mnemonic in ("HGMMA", "UBLKCP"):
        assert mnemonic in sass, mnemonic
    assert "HMMA.16816" not in sass  # no legacy mma.sync path


def test_no_cpu_fallback(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from adanerf_b200 import Renderer, AdnError
    from oracle import adanerf_oracle as orc
    with pytest.raises(AdnError) as e:
        Renderer(orc.SCENE_BARBERSHOP)
    assert e.value.status == 3  # ADN_ERR_NO_DEVICE


def test_product_package_does_not_import_oracle():
    pkg = os.path.join(ROOT, "adanerf_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert "import oracle" not in src and "from oracle" not in src, f


def test_build_is_idempotent_and_content_keyed():
    """build() decides by the content hash of the sources (sidecar .srchash), not by mtimes: calling it again -- or after a
    copy of the tree that touched every file -- must not start a compiler."""
    import os
    import __graft_entry__ as ge
    ge.build()
    before = {p: os.path.getmtime(p) for p in (ge.LIB, ge.MULTI_LIB, ge.VIEWER)}
    src = os.path.join(ge.CSRC, "api.cu")
    st = os.stat(src)
    try:
        os.utime(src, None)          # "newer than the library" by mtime
        ge.build()
    finally:
        os.utime(src, (st.st_atime, st.st_mtime))
    assert before == {p: os.path.getmtime(p) for p in before}
    assert not ge._stale(ge.LIB, ge.SOURCES + ge.HEADERS)
