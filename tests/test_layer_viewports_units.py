"""Audits of the layer-viewport kernel units (build.py VIEW_SOURCES), the checks tests/test_kernel_units.py makes of the other units,
each unit compiled once to PTX and once to a cubin with the shipped code-generation flags:

- packed contraction (DESIGN.md 2.3): no packed f32x2 op, and every mul.rn.f32 of the PTX survives as an FMUL in the SASS; the surplus
  is that of the unit the kernels come from (the FMULs of the IEEE division / reciprocal expansions of the final level's premin and
  slow paths);
- the CUDA-array units access their surfaces element by element, in zero mode;
- registers and spills: each kernel keeps the budget of the kernel it is a form of (prepare: 40 / 33 registers, the final upsample
  48), with no spill;
- completeness: each unit's kernel table holds every kernel the unit compiles to (meao_create loads the tables eagerly), and the emulator
  builds the same tables."""
import os
import re
import shutil
import subprocess
from concurrent.futures import ThreadPoolExecutor
from types import SimpleNamespace

import pytest

from emu import layer_views  # noqa: E402  (tests/ is on sys.path via conftest)
from miniengineao_b200.build import VIEW_SOURCES
from test_kernel_units import FLAGS, _entries  # noqa: E402  (the audit's flags and ptxas-log parser)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "miniengineao_b200", "csrc")

# unit -> (its kernels, FMUL minus mul.rn.f32, highest register count, kernel-name pattern)
UNITS = {
    "prepare_depth_array_views.cu": (5, 0, 40, r"prepare_depth_array_views_kernel"),
    "blur_upsample_array_views.cu": (2, 2, 48, r"blur_upsample_\w*array_views_kernel"),
    "prepare_depth_views.cu": (7, 0, 33, r"prepare_depth_low_views_kernel"),
    "blur_upsample_lin_views.cu": (6, 10, 48, r"blur_upsample_\w*lin_views_kernel"),
}


def test_every_view_unit_is_audited():
    assert sorted(UNITS) == sorted(VIEW_SOURCES)


@pytest.fixture(scope="module")
def units(tmp_path_factory):
    nvcc = "/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else shutil.which("nvcc")
    if not nvcc or not shutil.which("cuobjdump"):
        pytest.skip("nvcc / cuobjdump not available")
    tmp = str(tmp_path_factory.mktemp("view_units"))

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
        ptx = list(pool.map(compile_one, [(tu, "ptx") for tu in VIEW_SOURCES]))
        cubin = list(pool.map(compile_one, [(tu, "cubin") for tu in VIEW_SOURCES]))
    return {tu: SimpleNamespace(ptx=p, sass=c[0], entries=c[1]) for tu, p, c in zip(VIEW_SOURCES, ptx, cubin)}


@pytest.mark.parametrize("tu", VIEW_SOURCES)
def test_packed_mul_add_contractions_are_the_audited_ones(tu, units):
    p, s = units[tu].ptx, units[tu].sass
    assert "f32x2" not in p, tu
    assert not re.search(r"\b(FFMA2|FMUL2|FADD2)\b", s), tu
    n_mul = len(re.findall(r"\bmul\.rn\.f32\b", p))
    n_fmul = len(re.findall(r"\bFMUL\b", s))
    assert n_mul > 0 and n_fmul - n_mul == UNITS[tu][1], (tu, n_mul, n_fmul)


@pytest.mark.parametrize("tu", ["prepare_depth_array_views.cu", "blur_upsample_array_views.cu"])
def test_array_units_access_surfaces_element_by_element(tu, units):
    p = units[tu].ptx
    assert not re.search(r"\bsu(ld|st)\.b\.[a-z0-9]+\.v[24]", p), tu
    widths = set(re.findall(r"\bsu(?:ld|st)\.b\.[a-z0-9]+\.(b\d+)", p))
    assert widths and widths <= ({"b32", "b16"} if "prepare" in tu else {"b8"}), (tu, widths)
    assert ".trap" not in " ".join(re.findall(r"\bsu(?:ld|st)\.\S+", p)), tu


@pytest.mark.parametrize("tu", VIEW_SOURCES)
def test_registers_and_spills(tu, units):
    n, _, regs, pat = UNITS[tu]
    mine = [e for e in units[tu].entries if re.search(pat, e.name)]
    assert len(mine) == n, (tu, [e.name for e in mine])
    for e in mine:
        assert e.regs <= regs and e.spill_st == 0 and e.spill_ld == 0, vars(e)


def test_every_kernel_is_in_its_units_table(units):
    entries = {tu: len(re.findall(r"^\s*(?:\.\w+\s+)*\.entry\s", units[tu].ptx, re.M)) for tu in VIEW_SOURCES}
    assert entries == {tu: UNITS[tu][0] for tu in VIEW_SOURCES}
    assert layer_views.kernel_units() == entries
