"""Audits of the device-camera unit (build.py CAMERA_SOURCES: the camera tables derived on the device), compiled once to PTX and once to a
cubin with the shipped code-generation flags: no packed f32x2 op; every mul.rn.f32 of the PTX survives as an FMUL in the SASS, with no
surplus (the quotients are div.rn.f32, whose expansions add no FMUL here), so the products are the host planner's; spill-free with no
stack frame; and both .entry functions are in the unit's kernel table."""
import os
import re
import shutil
import subprocess
from types import SimpleNamespace

import pytest

from miniengineao_b200.build import CAMERA_SOURCES
from test_kernel_units import FLAGS, _entries  # noqa: E402  (the audit's flags and ptxas-log parser)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "miniengineao_b200", "csrc")
TU = "camera_tables.cu"
FMUL_SURPLUS = 0
KERNELS = {r"camera_tables_kernel": 1, r"camera_tables_mixed_kernel": 1}


def test_the_unit_is_audited():
    assert CAMERA_SOURCES == [TU]


@pytest.fixture(scope="module")
def unit(tmp_path_factory):
    nvcc = "/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else shutil.which("nvcc")
    if not nvcc or not shutil.which("cuobjdump"):
        pytest.skip("nvcc / cuobjdump not available")
    tmp = str(tmp_path_factory.mktemp("camera_unit"))
    ptx, cubin = os.path.join(tmp, "u.ptx"), os.path.join(tmp, "u.cubin")
    p = subprocess.run([nvcc] + FLAGS + ["-ptx", "-o", ptx, os.path.join(CSRC, TU)], capture_output=True, text=True)
    assert p.returncode == 0, p.stderr[-2000:]
    q = subprocess.run([nvcc] + FLAGS + ["-Xptxas", "-v", "-cubin", "-o", cubin, os.path.join(CSRC, TU)], capture_output=True, text=True)
    assert q.returncode == 0, q.stderr[-2000:]
    sass = subprocess.run(["cuobjdump", "-sass", cubin], capture_output=True, text=True, check=True).stdout
    return SimpleNamespace(ptx=open(ptx).read(), sass=sass, entries=_entries(q.stdout + q.stderr), log=q.stdout + q.stderr)


def test_no_packed_ops_and_every_product_kept(unit):
    assert "f32x2" not in unit.ptx
    assert not re.search(r"\b(FFMA2|FMUL2|FADD2)\b", unit.sass)
    n_mul = len(re.findall(r"\bmul\.rn\.f32\b", unit.ptx))
    n_fmul = len(re.findall(r"\bFMUL\b", unit.sass))
    assert n_mul > 0
    assert n_fmul - n_mul == FMUL_SURPLUS, (n_mul, n_fmul)
    # the one fused multiply-add is the atlas padding's fmaf, once per kernel
    assert len(re.findall(r"\bfma\.rn\.f32\b", unit.ptx)) == 2 * 2      # the perspective and the orthographic padding, in each kernel
    assert "div.rn.f32" in unit.ptx and "div.approx" not in unit.ptx and ".ftz" not in unit.ptx


def test_spill_free(unit):
    assert len(unit.entries) == sum(KERNELS.values())
    for pat, n in KERNELS.items():
        mine = [e for e in unit.entries if re.search(r"\d" + pat + r"E", e.name)]
        assert len(mine) == n, (pat, [e.name for e in unit.entries])
    for e in unit.entries:
        assert e.spill_st == 0 and e.spill_ld == 0, vars(e)
    assert not re.search(r"[1-9]\d* bytes stack frame", unit.log)


def test_every_kernel_is_in_its_units_table(unit):
    entries = len(re.findall(r"^\s*(?:\.\w+\s+)*\.entry\s", unit.ptx, re.M))
    src = open(os.path.join(CSRC, TU)).read()
    table = src[src.index("} kKernels = {"):src.index("}  // namespace\n")]
    listed = re.findall(r"camera_tables\w*_kernel", table)
    assert entries == len(listed) == sum(KERNELS.values())
    walk = src[src.index("kCameraTablesUnit"):]
    assert "kKernels.uniform" in walk and "kKernels.mixed" in walk
    # eager loading walks the unit (kernels.h kCameraKernelUnits, meao_api.cu meao_create)
    assert "&kCameraTablesUnit" in open(os.path.join(CSRC, "kernels.h")).read()
    assert "kCameraKernelUnits" in open(os.path.join(CSRC, "meao_api.cu")).read()
