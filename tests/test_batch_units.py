"""Audits of the batch kernel units (build.py BATCH_SOURCES), the checks tests/test_kernel_units.py makes of the other units,
each unit compiled once to PTX and once to a cubin with the shipped code-generation flags:

- packed contraction (DESIGN.md 2.3): no packed f32x2 op, and every mul.rn.f32 of the PTX survives as an FMUL in the SASS; the surplus
  is that of the unit the kernels come from (the FMULs of the IEEE division / reciprocal expansions of the final level's premin and
  slow paths);
- the CUDA-array units access their surfaces element by element, in zero mode;
- registers and spills: each kernel keeps the budget of its layer-viewport twin (prepare: 40 / 33 registers, the final upsample 48),
  with no spill, although its table is a 4 KB / 6 KB kernel parameter;
- the table is a __grid_constant__ parameter of that size, read in place (no local copy of it);
- completeness: each unit's kernel table holds every kernel the unit compiles to (meao_create loads the tables eagerly), and the emulator
  builds the same tables."""
import os
import re
import shutil
import subprocess
from concurrent.futures import ThreadPoolExecutor
from types import SimpleNamespace

import pytest

from emu import batch  # noqa: E402  (tests/ is on sys.path via conftest)
from miniengineao_b200.build import BATCH_SOURCES
from test_kernel_units import FLAGS, _entries  # noqa: E402  (the audit's flags and ptxas-log parser)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "miniengineao_b200", "csrc")

# unit -> (its kernels, FMUL minus mul.rn.f32, highest register count, kernel-name pattern)
UNITS = {
    "prepare_depth_array_batch.cu": (5, 0, 40, r"prepare_depth_array_batch_kernel"),
    "blur_upsample_array_batch.cu": (2, 2, 48, r"blur_upsample_\w*array_batch_kernel"),
    "prepare_depth_batch.cu": (7, 0, 33, r"prepare_depth_low_batch_kernel"),
    "blur_upsample_lin_batch.cu": (6, 10, 48, r"blur_upsample_\w*lin_batch_kernel"),
}


def test_every_batch_unit_is_audited():
    assert sorted(UNITS) == sorted(BATCH_SOURCES)


@pytest.fixture(scope="module")
def units(tmp_path_factory):
    nvcc = "/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else shutil.which("nvcc")
    if not nvcc or not shutil.which("cuobjdump"):
        pytest.skip("nvcc / cuobjdump not available")
    tmp = str(tmp_path_factory.mktemp("batch_units"))

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
        ptx = list(pool.map(compile_one, [(tu, "ptx") for tu in BATCH_SOURCES]))
        cubin = list(pool.map(compile_one, [(tu, "cubin") for tu in BATCH_SOURCES]))
    return {tu: SimpleNamespace(ptx=p, sass=c[0], entries=c[1]) for tu, p, c in zip(BATCH_SOURCES, ptx, cubin)}


@pytest.mark.parametrize("tu", BATCH_SOURCES)
def test_packed_mul_add_contractions_are_the_audited_ones(tu, units):
    p, s = units[tu].ptx, units[tu].sass
    assert "f32x2" not in p, tu
    assert not re.search(r"\b(FFMA2|FMUL2|FADD2)\b", s), tu
    n_mul = len(re.findall(r"\bmul\.rn\.f32\b", p))
    n_fmul = len(re.findall(r"\bFMUL\b", s))
    assert n_mul > 0 and n_fmul - n_mul == UNITS[tu][1], (tu, n_mul, n_fmul)


@pytest.mark.parametrize("tu", ["prepare_depth_array_batch.cu", "blur_upsample_array_batch.cu"])
def test_array_units_access_surfaces_element_by_element(tu, units):
    p = units[tu].ptx
    assert not re.search(r"\bsu(ld|st)\.b\.[a-z0-9]+\.v[24]", p), tu
    widths = set(re.findall(r"\bsu(?:ld|st)\.b\.[a-z0-9]+\.(b\d+)", p))
    assert widths and widths <= ({"b32", "b16"} if "prepare" in tu else {"b8"}), (tu, widths)
    assert ".trap" not in " ".join(re.findall(r"\bsu(?:ld|st)\.\S+", p)), tu


@pytest.mark.parametrize("tu", BATCH_SOURCES)
def test_registers_and_spills(tu, units):
    n, _, regs, pat = UNITS[tu]
    mine = [e for e in units[tu].entries if re.search(pat, e.name)]
    assert len(mine) == n, (tu, [e.name for e in mine])
    for e in mine:
        assert e.regs <= regs and e.spill_st == 0 and e.spill_ld == 0, vars(e)


def test_every_kernel_is_in_its_units_table(units):
    entries = {tu: len(re.findall(r"^\s*(?:\.\w+\s+)*\.entry\s", units[tu].ptx, re.M)) for tu in BATCH_SOURCES}
    assert entries == {tu: UNITS[tu][0] for tu in BATCH_SOURCES}
    assert batch.kernel_units() == entries


# unit -> the bytes of its table parameter (kernels.h BatchArrays / BatchPointers)
TABLE_BYTES = {"prepare_depth_array_batch.cu": 4096, "blur_upsample_array_batch.cu": 4096, "prepare_depth_batch.cu": 6144,
               "blur_upsample_lin_batch.cu": 6144}


@pytest.mark.parametrize("tu", BATCH_SOURCES)
def test_table_is_a_grid_constant_parameter_read_in_place(tu, units):
    p = units[tu].ptx
    entries = re.split(r"\.entry\s", p)[1:]
    assert len(entries) == UNITS[tu][0], tu
    for e in entries:
        params = re.findall(r"\.param\s+\.align\s+(\d+)\s+\.b8\s+(\w+)\[(\d+)\]", e.split(")", 1)[0])
        assert any(int(n) == TABLE_BYTES[tu] for _, _, n in params), (tu, params)
    # the table stays in the parameter bank: no local-memory copy of it
    assert not re.search(r"\.local\s+\.align\s+\d+\s+\.b8\s+\w+\[(4096|6144)\]", p), tu
