"""Audits of the per-layer projection kernel units (build.py MIXED_SOURCES: a layered frame whose layers mix both projections), each
compiled once to PTX and once to a cubin with the shipped code-generation flags: no packed f32x2 op; registers within the budget of the
orthographic twin each mirrors (prepare 40 / low-only 33, render 40 = MEAO_REN_MINB 6, fused final upsample 48), and the CUDA-array
prepare, which holds both linearisations, bounded at 5 CTAs per SM (48) like its twin; no spill anywhere; the 8 KB LayerProjections
parameter in every kernel; and every .entry of a unit is in its kernel table (34 kernels)."""
import os
import re
import shutil
import subprocess
from concurrent.futures import ThreadPoolExecutor
from types import SimpleNamespace

import pytest

from miniengineao_b200.build import MIXED_SOURCES
from test_kernel_units import FLAGS, _entries  # noqa: E402  (the audit's flags and ptxas-log parser)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "miniengineao_b200", "csrc")

# unit -> {kernel-name pattern: (kernels, highest register count)}
UNITS = {
    "prepare_depth_mixed_layered.cu": {r"prepare_depth_mixed_layered_kernel": (6, 40), r"prepare_depth_low_mixed_layered_kernel": (6, 33)},
    "prepare_depth_array_mixed.cu": {r"prepare_depth_array_mixed_kernel": (4, 48)},
    "render_ao_mixed_layered.cu": {r"render_ao_mixed_layered_kernel": (12, 40)},
    "blur_upsample_lin_mixed.cu": {r"blur_upsample_\w*lin_mixed_kernel": (6, 48)},
}


def test_every_mixed_unit_is_audited():
    assert sorted(UNITS) == sorted(MIXED_SOURCES)
    assert sum(n for u in UNITS.values() for n, _ in u.values()) == 34


@pytest.fixture(scope="module")
def units(tmp_path_factory):
    nvcc = "/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else shutil.which("nvcc")
    if not nvcc or not shutil.which("cuobjdump"):
        pytest.skip("nvcc / cuobjdump not available")
    tmp = str(tmp_path_factory.mktemp("mixed_units"))

    def compile_one(job):
        tu, kind = job
        out = os.path.join(tmp, tu + "." + kind)
        extra = ["-ptx"] if kind == "ptx" else ["-Xptxas", "-v", "-cubin"]
        p = subprocess.run([nvcc] + FLAGS + extra + ["-o", out, os.path.join(CSRC, tu)], capture_output=True, text=True)
        assert p.returncode == 0, (tu, p.stderr[-2000:])
        if kind == "ptx":
            return open(out).read()
        return subprocess.run(["cuobjdump", "-sass", out], capture_output=True, text=True, check=True).stdout, _entries(p.stdout + p.stderr)

    with ThreadPoolExecutor(max_workers=os.cpu_count() or 1) as pool:
        ptx = list(pool.map(compile_one, [(tu, "ptx") for tu in MIXED_SOURCES]))
        cubin = list(pool.map(compile_one, [(tu, "cubin") for tu in MIXED_SOURCES]))
    return {tu: SimpleNamespace(ptx=p, sass=c[0], entries=c[1]) for tu, p, c in zip(MIXED_SOURCES, ptx, cubin)}


@pytest.mark.parametrize("tu", MIXED_SOURCES)
def test_no_packed_ops(tu, units):
    assert "f32x2" not in units[tu].ptx, tu
    assert not re.search(r"\b(FFMA2|FMUL2|FADD2)\b", units[tu].sass), tu


@pytest.mark.parametrize("tu", MIXED_SOURCES)
def test_registers_and_spills(tu, units):
    seen = 0
    for pat, (n, regs) in UNITS[tu].items():
        mine = [e for e in units[tu].entries if re.search(r"\d" + pat, e.name)]
        assert len(mine) == n, (tu, pat, [e.name for e in mine])
        for e in mine:
            assert e.regs <= regs and e.spill_st == 0 and e.spill_ld == 0, vars(e)
        seen += n
    assert seen == len(units[tu].entries), tu


@pytest.mark.parametrize("tu", MIXED_SOURCES)
def test_projection_table_is_a_parameter(tu, units):
    """Every kernel takes the 8 KB LayerProjections table by value (.param .align 4 .b8 ..[8192])."""
    entries = re.findall(r"\.entry\s+(\w+)\(([^)]*)\)", units[tu].ptx)
    assert entries
    for name, params in entries:
        assert re.search(r"\.param \.align \d+ \.b8 \w+\[8192\]", params), name


@pytest.mark.parametrize("tu", MIXED_SOURCES)
def test_every_kernel_is_in_its_units_table(tu, units):
    entries = len(re.findall(r"^\s*(?:\.\w+\s+)*\.entry\s", units[tu].ptx, re.M))
    assert entries == sum(n for n, _ in UNITS[tu].values())
    src = open(os.path.join(CSRC, tu)).read()
    table = src[src.index("kKernels"):src.index("}  // namespace\n")]
    slots = len(re.findall(r"MEAO_PREPARE_SLOTS_RAW\((\w+), MEAO_SLOT\)", table)) * 6 + \
        len(re.findall(r"MEAO_PREPARE_SLOTS_RAW\((\w+), MEAO_NO_SLOT\)", table)) * 4 + \
        len(re.findall(r"MEAO_RENDER_SLOTS\(", table)) * 12 + len(re.findall(r"MEAO_LIN_SLOTS\(", table)) * 3
    assert slots == entries, (tu, slots, entries)
