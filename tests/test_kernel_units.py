"""Audits of every kernel translation unit (build.py SOURCES less the context, meao_api.cu), each compiled once to PTX and once to
a cubin with the shipped code-generation flags:

- packed contraction (DESIGN.md 2.3): the arithmetic contract with the oracle is that a*b+c is fused only where the source says
  fmaf(); -fmad=false and the _rn intrinsics keep nvcc and ptxas from fusing on their own, and the kernels' two-lane helpers
  (ffma2 / fmul2 / fadd2, common.cuh) must stay lane-wise scalar: a packed f32x2 form does not exist on sm_90a, and where it does
  exist ptxas contracts a packed mul -> add even with explicit .rn.  No packed op may appear, and every mul.rn.f32 of the PTX must
  survive as an FMUL in the SASS (a contraction removes one).  The expected surplus is the audited one (FMULs of the IEEE division /
  reciprocal expansions); a change must be looked at before the numbers here are updated.
- the CUDA-array units' surface accesses, and the registers and spills of the kernels tuned against a budget;
- completeness: each unit's kernel table (kernels.h) holds every kernel the unit compiles to.  meao_create loads the kernels eagerly
  by walking the tables, and a kernel left out would load lazily on its first launch -- behind a spinning band exchange kernel, that
  load waits until the exchange times out.
"""
import os
import re
import shutil
import subprocess
from concurrent.futures import ThreadPoolExecutor
from types import SimpleNamespace

import pytest

from emu import emu  # noqa: E402  (tests/ is on sys.path via conftest)
from miniengineao_b200.build import SOURCES

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "miniengineao_b200", "csrc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-fmad=false"]
UNITS = [s for s in SOURCES if s != "meao_api.cu"]

# translation unit -> FMUL (SASS) minus mul.rn.f32 (PTX): multiplies ptxas adds when it expands div.rn / rcp.rn
FMUL_SURPLUS = {
    "prepare_depth.cu": 0, "prepare_depth_layered.cu": 0, "prepare_depth_array.cu": 0,
    "render_ao.cu": 0, "render_ao_layered.cu": 0,
    "blur_upsample.cu": 6, "blur_upsample_layered.cu": 6,      # the premin kernels: 2 in the final level's, 4 in the blend levels'
    "blur_upsample_lin.cu": 22,     # its 12 kernels
    "blur_upsample_array.cu": 2,    # the two final-level kernels
    "selftest.cu": 0, "halo.cu": 0, "band_exchange.cu": 0, "composite.cu": 0, "debug_view.cu": 0,
}
NO_MUL = {"halo.cu", "band_exchange.cu"}        # copies only: no mul.rn.f32 to audit

# translation unit -> its kernels (.entry functions of its PTX): the instantiations its kernel table lists (kernels.h MEAO_*_SLOTS)
ENTRIES = {
    "prepare_depth.cu": 14, "prepare_depth_layered.cu": 14, "prepare_depth_array.cu": 5,
    "render_ao.cu": 13, "render_ao_layered.cu": 12,
    "blur_upsample.cu": 4, "blur_upsample_layered.cu": 4, "blur_upsample_array.cu": 2, "blur_upsample_lin.cu": 12,
    "selftest.cu": 1, "halo.cu": 1, "band_exchange.cu": 1, "composite.cu": 2, "debug_view.cu": 3,
}

# translation unit -> (kernel-name pattern, number of kernels): the pitch replaces the W multiplier and must not cost a spill
SPILL_FREE = {"blur_upsample_lin.cu": (r"blur_upsample_\w*lin\w*_kernel", 12), "prepare_depth.cu": (r"prepare_depth_\w*kernel", 14),
              "prepare_depth_layered.cu": (r"prepare_depth_\w*kernel", 14)}

# kernels that read a per-layer camera value: (kernel name prefix) -> (translation unit, the highest register count and spill bytes
# allowed); the counts before per-layer cameras, except where noted in DESIGN.md 2.9 (the occupancy they allow is unchanged)
LIMITS = {"render_ao_layered_kernel": ("render_ao_layered.cu", 40, 0), "prepare_depth_layered_kernel": ("prepare_depth_layered.cu", 40, 0),
          "prepare_depth_low_layered_kernel": ("prepare_depth_layered.cu", 33, 0), "prepare_depth_array_kernel": ("prepare_depth_array.cu", 40, 0),
          "blur_upsample_lin_layered_kernel": ("blur_upsample_lin.cu", 48, 0)}


def _entries(ptxas_log: str) -> list:
    """-Xptxas -v output -> one (name, registers, spill store bytes, spill load bytes) per entry function (not per device function)"""
    out, cur = [], None
    for line in ptxas_log.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            out.append(SimpleNamespace(name=m.group(1), regs=None, spill_st=None, spill_ld=None))
            cur = out[-1]
            continue
        m = re.search(r"Function properties for (\w+)", line)
        if m:
            cur = out[-1] if out and out[-1].name == m.group(1) else None
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur:
            cur.spill_st, cur.spill_ld = int(m.group(1)), int(m.group(2))
        m = re.search(r"Used (\d+) registers", line)
        if m and cur:
            cur.regs = int(m.group(1))
    return out


@pytest.fixture(scope="module")
def units(tmp_path_factory):
    """unit -> .ptx (PTX text), .sass (cuobjdump -sass of its cubin), .entries (_entries of its ptxas log); compiled in parallel"""
    nvcc = "/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else shutil.which("nvcc")
    if not nvcc or not shutil.which("cuobjdump"):
        pytest.skip("nvcc / cuobjdump not available")
    tmp = str(tmp_path_factory.mktemp("kernel_units"))

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
        ptx = pool.map(compile_one, [(tu, "ptx") for tu in UNITS])
        cubin = pool.map(compile_one, [(tu, "cubin") for tu in UNITS])
        return {tu: SimpleNamespace(ptx=p, sass=c[0], entries=c[1]) for tu, p, c in zip(UNITS, ptx, cubin)}


@pytest.mark.parametrize("tu", UNITS)
def test_packed_mul_add_contractions_are_the_audited_ones(tu, units):
    p, s = units[tu].ptx, units[tu].sass
    assert "f32x2" not in p, tu
    assert not re.search(r"\b(FFMA2|FMUL2|FADD2)\b", s), tu
    n_mul = len(re.findall(r"\bmul\.rn\.f32\b", p))
    n_fmul = len(re.findall(r"\bFMUL\b", s))
    assert n_mul > 0 or tu in NO_MUL, tu
    assert n_fmul - n_mul == FMUL_SURPLUS[tu], (tu, n_mul, n_fmul)


@pytest.mark.parametrize("tu", ["prepare_depth_array.cu", "blur_upsample_array.cu"])
def test_array_units_access_surfaces_element_by_element(tu, units):
    """32- / 16-bit surface loads, 8-bit stores, never a vector form, every access in zero mode (no .trap)"""
    p = units[tu].ptx
    assert not re.search(r"\bsu(ld|st)\.b\.[a-z0-9]+\.v[24]", p), tu
    widths = set(re.findall(r"\bsu(?:ld|st)\.b\.[a-z0-9]+\.(b\d+)", p))
    assert widths, tu
    assert widths <= ({"b32", "b16"} if "prepare" in tu else {"b8"}), (tu, widths)
    assert ".trap" not in " ".join(re.findall(r"\bsu(?:ld|st)\.\S+", p)), tu


@pytest.mark.parametrize("tu", sorted(SPILL_FREE))
def test_pitched_kernels_do_not_spill(tu, units):
    """the fused final-level kernels (48-register cap) and both prepare forms: 0 bytes of spill each"""
    pat, n = SPILL_FREE[tu]
    mine = [e for e in units[tu].entries if re.search(pat, e.name)]
    assert len(mine) == n, (tu, [e.name for e in mine])
    assert all(e.spill_st == 0 and e.spill_ld == 0 for e in mine), [vars(e) for e in mine]


@pytest.mark.parametrize("kernel", sorted(LIMITS))
def test_per_layer_kernels_keep_registers_and_spills(kernel, units):
    tu, regs, spill = LIMITS[kernel]
    mine = [e for e in units[tu].entries if re.search(r"\d+%sI" % kernel, e.name)]
    assert mine, kernel
    for e in mine:
        assert e.regs <= regs and e.spill_st <= spill, vars(e)


def test_every_kernel_is_in_its_units_table(units):
    """The .entry functions of each unit's PTX against the kernel count of its table, as the emulator builds the units (all but the
    GPU self test, whose table is its one kernel).  The counts are pinned too: a templated kernel left out of its table is not
    instantiated at all, so it would vanish from the PTX and the table alike."""
    entries = {tu: len(re.findall(r"^\s*(?:\.\w+\s+)*\.entry\s", units[tu].ptx, re.M)) for tu in UNITS}
    assert entries == ENTRIES
    tables = emu.kernel_units()
    assert set(tables) == set(emu.build_emu.KERNELS)
    assert tables == {tu: entries[tu] for tu in tables}
