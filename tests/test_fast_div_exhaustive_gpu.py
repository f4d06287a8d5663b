"""Exhaustive checks of the fast-division building blocks the kernels run (csrc/common.cuh, csrc/blur_upsample_device.inc).

tests/gpu_probes/fast_div_probe.cu includes those sources as the kernels do and compares, against float64 statements of their
contracts: the range predicates in_safe_range / in_safe_range_neg and the bilateral pair guard on all 2^32 bit patterns; rcp_fast and
both lanes of rcp2_fast_neg on every in-range operand; div_fast and div2_fast_neg on every in-range denominator for the bilateral
numerators 1, 3, 9 and on a seeded sample of in-range pairs; bilateral2 against the scalar IEEE bilateral on adversarial operands
(exact ties, f16 depths, the edges of the host-proven tolerance range, AO codes 0 / 1 / 255).  The emulator's MUFU.RCP is correctly
rounded, so only the GPU run proves the approximation path; the predicate part also runs on the CPU, as a host build of the probe."""
import os
import re
import shutil
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "miniengineao_b200", "csrc")
PROBE = os.path.join(HERE, "gpu_probes", "fast_div_probe.cu")
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-fmad=false"]     # the flags libmeao is built with
IN_RANGE = 120 << 23            # positive normal floats in [2^-60, 2^60): biased exponents 67 .. 186


def _parse(out):
    res = {m[0]: (int(m[1]), int(m[2])) for m in re.findall(r"^RESULT (\S+) checked=(\d+) mismatches=(\d+)$", out, re.M)}
    counts = {m[0]: int(m[1]) for m in re.findall(r"^COUNT (\S+) (\d+)$", out, re.M)}
    return res, counts


def _check_part1(res, counts):
    assert res["in_safe_range"] == (1 << 32, 0), res["in_safe_range"]
    assert res["in_safe_range_neg"] == (1 << 32, 0), res["in_safe_range_neg"]
    # every pattern with the sign bit set (2^31) and every positive NaN (2^23 - 1)
    assert res["pair_guard"] == ((1 << 31) + (1 << 23) - 1, 0), res["pair_guard"]
    assert counts["in_range"] == IN_RANGE


def test_guard_predicates_on_every_bit_pattern_host_build(tmp_path):
    """Part 1 of the probe as a host program (-DMEAO_EMULATE): the predicates are integer bit tricks, identical on both sides."""
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("g++ not available")
    exe = str(tmp_path / "fast_div_probe_host")
    subprocess.check_call([gxx, "-std=c++17", "-O2", "-ffp-contract=off", "-DMEAO_EMULATE", "-I", os.path.join(HERE, "emu"), "-I", CSRC,
                           "-x", "c++", PROBE, "-o", exe, "-pthread"])
    out = subprocess.run([exe], capture_output=True, text=True, check=True, timeout=600).stdout
    res, counts = _parse(out)
    _check_part1(res, counts)


@pytest.mark.gpu
def test_fast_division_building_blocks_exhaustive_on_the_gpu(tmp_path):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    nvcc = "/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else shutil.which("nvcc")
    if not nvcc:
        pytest.skip("nvcc not available")
    exe = str(tmp_path / "fast_div_probe")
    subprocess.check_call([nvcc] + NVCC_FLAGS + ["-I", CSRC, PROBE, "-o", exe])
    p = subprocess.run([exe], capture_output=True, text=True, timeout=1800)
    print(p.stdout)
    assert p.returncode == 0, p.stdout + p.stderr
    res, counts = _parse(p.stdout)
    _check_part1(res, counts)
    for name in ("rcp_fast", "rcp2_fast_neg.x", "rcp2_fast_neg.y", "ieee_rcp") + \
            tuple(f"{f}.a{a}" for a in (1, 3, 9) for f in ("div_fast", "div2_fast_neg.x", "div2_fast_neg.y")):
        assert res[name] == (IN_RANGE, 0), (name, res[name])
    assert res["ieee_div.a1_3_9"] == (3 * IN_RANGE, 0)
    n = res["div_fast.random"][0]
    assert n > (1 << 30), n                # draws of two pairs: both quotients are in range in about 56 % of the 2^31 draws
    for name in ("div_fast.random", "div2_fast_neg.x.random", "div2_fast_neg.y.random", "ieee_div.random"):
        assert res[name] == (n, 0), (name, res[name])
    for blend in (0, 1):
        checked, bad = res[f"bilateral2.blend{blend}"]
        fallback = counts[f"bilateral2.blend{blend}.fallback"]
        assert bad == 0, (blend, checked, bad)
        assert checked + fallback == 1 << 32 and checked > (1 << 31) and fallback > 0, (blend, checked, fallback)
