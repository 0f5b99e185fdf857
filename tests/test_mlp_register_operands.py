"""CPU-side check of mlp_kernel<1>'s register-resident activations (the shading net, and the plain bf16 sampling net).
Each hidden layer's bf16 output stays in the consumer threads' registers and feeds the next layer's MMAs as wgmma's
register A operand.  That only pays if the compiler
keeps those 64 fragment registers in registers: a fragment array demoted to local memory (LDL / STL), a spill, or a
wgmma that ptxas serialises because its register operands are touched while it runs would each cost more than the
shared-memory round trip the register operand replaces."""
import os
import re
import shutil
import subprocess

import pytest

# mlp_kernel<1, true> runs the fused input encoder, whose accurate sincosf keeps a 28-byte Payne-Hanek reduction table on
# the stack for huge arguments: its only local memory.  A fragment array in local memory would take 256 bytes.
ENCODER_STACK_BYTES = 32


def _mlp_sass():
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
    assert len(kernels) == 3, sorted(kernels)
    return kernels


def _instantiation(name):
    m = re.search(r"mlp_kernelILi(\d)ELb(\d)E", name)
    assert m, name
    return int(m.group(1)), bool(int(m.group(2)))


def test_shading_hidden_layers_multiply_from_registers():
    for name, body in _mlp_sass().items():
        nsplit, _ = _instantiation(name)
        hgmma = re.findall(r"\sHGMMA\.64x128x16\S*\s+([^;]*);", body)
        register_a = [ops for ops in hgmma if re.match(r"R\d+, R\d+, gdesc\[", ops)]
        if nsplit == 1:
            # two N halves x at most four hidden K blocks x four K steps, unrolled: the fragment index is a constant
            assert len(register_a) >= 16, (name, hgmma[:4])
        else:
            assert not register_a, (name, register_a[:4])   # the sampling net's hi / lo split stays in shared memory


def test_mlp_kernels_use_no_local_memory():
    for name, body in _mlp_sass().items():
        _, enc = _instantiation(name)
        local = re.findall(r"\s((?:LDL|STL)\S*)", body)
        if not enc:
            assert not local, (name, local[:5])


def test_ptxas_reports_no_spills_and_no_serialised_wgmma(tmp_path):
    import __graft_entry__ as g
    nvcc = g._nvcc()
    if os.path.isabs(nvcc) and not os.path.exists(nvcc) or not os.path.isabs(nvcc) and not shutil.which(nvcc):
        pytest.skip("nvcc not available")
    flags = [f for f in g.NVCC_FLAGS if f != "-shared"]
    r = subprocess.run([nvcc] + flags + ["-c", "-Xptxas", "-v", "-o", str(tmp_path / "mlp.o"), "mlp.cu"],
                       cwd=g.CSRC, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    log = r.stdout + r.stderr
    serialised = [line for line in log.splitlines() if "mlp_kernel" in line and ("C7510" in line or "serializ" in line.lower())]
    assert not serialised, serialised[:3]
    reports = []
    for part in log.split("Compiling entry function '")[1:]:
        name = part.split("'", 1)[0]
        if "mlp_kernel" in name:
            reports.append((name,) + re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", part).groups())
    assert len(reports) == 3, log[-2000:]
    for name, stack, spill_st, spill_ld in reports:
        _, enc = _instantiation(name)
        assert int(spill_st) == 0 and int(spill_ld) == 0, (name, spill_st, spill_ld)
        assert int(stack) <= (ENCODER_STACK_BYTES if enc else 0), (name, stack)
