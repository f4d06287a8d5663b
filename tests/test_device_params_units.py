"""Audits of the device-parameter units (build.py PARAM_SOURCES: the parameter stage and the three *_params_layered render twins), each
compiled once to PTX and once to a cubin with the shipped code-generation flags: no packed f32x2 op; every mul.rn.f32 of the PTX survives
as an FMUL in the SASS, with no surplus; the parameter stage's quotient is an IEEE div.rn.f32 without flush-to-zero; the twins stay within
the render's register cap (__launch_bounds__(256, 6): 40 registers) and every kernel is spill-free with no stack frame; every .entry is in
its unit's kernel table, which eager loading walks.  And the hooks the twins are built from are off in the existing render units: the
macro does not leak into them.  That the existing kernels' SASS is unchanged is a comparison of two library builds, which this audit
cannot make without the parent's sources (scripts/sass_diff.py, DESIGN.md 2.21)."""
import os
import re
import shutil
import subprocess
from concurrent.futures import ThreadPoolExecutor
from types import SimpleNamespace

import pytest

from miniengineao_b200.build import PARAM_SOURCES
from test_kernel_units import FLAGS, _entries  # noqa: E402  (the audit's flags and ptxas-log parser)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "miniengineao_b200", "csrc")
# unit -> (kernel-name pattern, kernels, FMUL minus mul.rn.f32)
UNITS = {
    "render_params.cu": (r"render_params_kernel", 1, 0),
    "render_ao_params_layered.cu": (r"render_ao_params_layered_kernel", 12, 0),
    "render_ao_ortho_params_layered.cu": (r"render_ao_ortho_params_layered_kernel", 12, 0),
    "render_ao_mixed_params_layered.cu": (r"render_ao_mixed_params_layered_kernel", 12, 0),
}
REGISTER_CAP = 40           # render_ao_kernel.inc: __launch_bounds__(256, MEAO_REN_MINB = 6) on 64 K registers
EXISTING_RENDER_UNITS = ["render_ao.cu", "render_ao_layered.cu", "render_ao_ortho.cu", "render_ao_ortho_layered.cu", "render_ao_mixed_layered.cu"]


def _nvcc():
    nvcc = "/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else shutil.which("nvcc")
    if not nvcc or not shutil.which("cuobjdump"):
        pytest.skip("nvcc / cuobjdump not available")
    return nvcc


def test_the_units_are_audited():
    assert PARAM_SOURCES == list(UNITS)


@pytest.fixture(scope="module")
def units(tmp_path_factory):
    nvcc = _nvcc()
    tmp = str(tmp_path_factory.mktemp("param_units"))

    def compile_one(tu):
        ptx, cubin = os.path.join(tmp, tu + ".ptx"), os.path.join(tmp, tu + ".cubin")
        p = subprocess.run([nvcc] + FLAGS + ["-ptx", "-o", ptx, os.path.join(CSRC, tu)], capture_output=True, text=True)
        assert p.returncode == 0, (tu, p.stderr[-2000:])
        q = subprocess.run([nvcc] + FLAGS + ["-Xptxas", "-v", "-cubin", "-o", cubin, os.path.join(CSRC, tu)], capture_output=True, text=True)
        assert q.returncode == 0, (tu, q.stderr[-2000:])
        sass = subprocess.run(["cuobjdump", "-sass", cubin], capture_output=True, text=True, check=True).stdout
        return SimpleNamespace(ptx=open(ptx).read(), sass=sass, entries=_entries(q.stdout + q.stderr), log=q.stdout + q.stderr)

    with ThreadPoolExecutor(max_workers=len(UNITS)) as pool:
        return dict(zip(UNITS, pool.map(compile_one, UNITS)))


@pytest.mark.parametrize("tu", list(UNITS))
def test_no_packed_ops_and_every_product_kept(tu, units):
    u = units[tu]
    assert "f32x2" not in u.ptx
    assert not re.search(r"\b(FFMA2|FMUL2|FADD2)\b", u.sass)
    n_mul = len(re.findall(r"\bmul\.rn\.f32\b", u.ptx))
    n_fmul = len(re.findall(r"\bFMUL\b", u.sass))
    assert n_fmul - n_mul == UNITS[tu][2], (tu, n_mul, n_fmul)
    if tu == "render_params.cu":
        # -1 / thickness_modifier: the IEEE quotient, subnormal operands kept (the host planner's bits)
        assert n_mul == 0 and "div.rn.f32" in u.ptx and "div.approx" not in u.ptx and ".ftz" not in u.ptx
    else:
        assert n_mul > 0


@pytest.mark.parametrize("tu", list(UNITS))
def test_registers_and_spills(tu, units):
    pat, n, _ = UNITS[tu]
    u = units[tu]
    assert len(u.entries) == n, (tu, [e.name for e in u.entries])
    assert all(re.search(r"\d" + pat + r"[IE]", e.name) for e in u.entries), [e.name for e in u.entries]
    for e in u.entries:
        assert e.spill_st == 0 and e.spill_ld == 0, vars(e)
        assert e.regs <= REGISTER_CAP, vars(e)
    assert not re.search(r"[1-9]\d* bytes stack frame", u.log)


@pytest.mark.parametrize("tu", list(UNITS))
def test_every_kernel_is_in_its_units_table(tu, units):
    pat, n, _ = UNITS[tu]
    entries = len(re.findall(r"^\s*(?:\.\w+\s+)*\.entry\s", units[tu].ptx, re.M))
    src = open(os.path.join(CSRC, tu)).read()
    table = src[src.index("kKernels"):src.index("}  // namespace\n")]
    if tu == "render_params.cu":
        assert re.findall(r"render_params_kernel", table) == ["render_params_kernel"]
        assert "kKernels.derive" in src[src.index("kRenderParamsUnit"):]
    else:
        assert re.search(r"kKernels\[kRenderSlots\] =\s+MEAO_RENDER_SLOTS\(" + pat + r"\)", table), tu
        assert "walk_kernels(load, kKernels)" in src[src.rindex("const KernelUnit"):]
    assert entries == n
    # eager loading walks every unit (kernels.h kParamKernelUnits, meao_api.cu meao_create)
    kernels_h = open(os.path.join(CSRC, "kernels.h")).read()
    unit = re.search(r"const KernelUnit (k\w+Unit) = \{\"" + re.escape(tu) + '"', src).group(1)
    lst = kernels_h[kernels_h.index("kParamKernelUnits[] = {"):]
    assert "&" + unit in lst[:lst.index("};")], unit
    assert "kParamKernelUnits" in open(os.path.join(CSRC, "meao_api.cu")).read()


def _at_zero(text: str) -> str:
    """text with every `#if MEAO_DEVICE_PARAMS` / `#if !MEAO_DEVICE_PARAMS` block (optionally with `#else`) resolved as for the macro at 0."""
    out, state = [], None            # state: None outside a block; else (keep_now, negated)
    for line in text.splitlines(keepends=True):
        s = line.strip()
        if state is None and s in ("#if MEAO_DEVICE_PARAMS", "#if !MEAO_DEVICE_PARAMS"):
            state = s.startswith("#if !")
            continue
        if state is not None and s == "#else":
            state = not state
            continue
        if state is not None and s == "#endif":
            state = None
            continue
        if state is None or state:
            out.append(line)
    return "".join(out)


def test_the_hooks_are_off_in_the_existing_render_units(tmp_path):
    """Each existing render unit preprocesses to the same source with the hooked .inc files as with copies whose MEAO_DEVICE_PARAMS blocks
    are resolved at 0.  This guards the macro, not the code generation: it fails when an existing unit or a header it includes defines
    MEAO_DEVICE_PARAMS, or when a hook is written in a form other than the `#if MEAO_DEVICE_PARAMS` / `#if !MEAO_DEVICE_PARAMS` blocks
    (whose resolution at 0 this test spells out by hand, as the preprocessor does for an undefined macro)."""
    nvcc = _nvcc()
    plain = tmp_path / "csrc"
    shutil.copytree(CSRC, plain)
    hooked = 0
    for inc in ("render_ao_kernel.inc", "render_ao_sample.inc"):
        text = (plain / inc).read_text()
        hooked += len(re.findall(r"^\s*#if !?MEAO_DEVICE_PARAMS$", text, re.M))
        (plain / inc).write_text(_at_zero(text))
        assert not re.search(r"^\s*#.*MEAO_DEVICE_PARAMS", (plain / inc).read_text(), re.M)
    assert hooked >= 4

    def pre(d, tu):
        p = subprocess.run([nvcc] + FLAGS + ["-E", "-Xcompiler", "-P", os.path.join(d, tu)], capture_output=True, text=True)
        assert p.returncode == 0, (tu, p.stderr[-2000:])
        return p.stdout

    for tu in EXISTING_RENDER_UNITS:
        assert pre(CSRC, tu) == pre(str(plain), tu), tu
