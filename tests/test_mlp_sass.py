"""CPU-side check of the MLP kernels' machine code: the epilogue reads its biases and head weights and writes the next
layer's activations in shared memory, and those accesses must compile to LDS / STS.  A generic LD.E / ST.E there (a
pointer the compiler can no longer place in the shared state space) nearly doubles the shading MLP's time on the H100."""
import os
import re
import shutil
import subprocess

import pytest


def test_mlp_kernels_use_no_generic_loads_or_stores():
    import __graft_entry__ as g
    g.build()
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", g.LIB], capture_output=True, text=True).stdout
    kernels = {}
    for part in re.split(r"\n\s+Function : ", sass)[1:]:
        name = part.split("\n", 1)[0].strip()
        if "mlp_kernel" in name:
            kernels[name] = part
    assert len(kernels) == 3, sorted(kernels)   # <2,false>, <1,false>, <1,true>
    for name, body in kernels.items():
        generic = re.findall(r"\s((?:LD|ST)\.E\S*)", body)
        assert not generic, (name, generic[:5])
        assert re.search(r"\sLDS\.64\s", body), name
