"""CPU tests of the C-ABI library: it loads without a GPU or driver, exports every symbol include/meao.h
declares, fails LOUDLY when asked to compute without a device, and its host-side planner (constants,
geometry, band/halo ranges) agrees with the oracle's restatement of AmbientOcclusion.cs."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from miniengineao_b200 import AmbientOcclusion, Camera, MeaoError
from miniengineao_b200 import _native as N
from oracle.oracle import Oracle

import harness

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_functions():
    src = open(os.path.join(ROOT, "include", "meao.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    names = set(re.findall(r"\b(meao_[a-z0-9_]+)\s*\(", src))
    return sorted(names)


def test_library_exports_every_declared_symbol():
    lib = N.lib()
    decl = _declared_functions()
    assert len(decl) >= 35
    for name in decl:
        assert hasattr(lib, name), f"{name} declared in include/meao.h but not exported"
        assert name in N.SIGNATURES, f"{name} has no ctypes signature in _native.py"
    out = subprocess.run(["nm", "-D", "--defined-only", N.LIB_PATH], capture_output=True, text=True).stdout
    exported = set(re.findall(r" T (meao_[a-z0-9_]+)", out))
    assert set(decl) <= exported
    assert lib.meao_abi_version() == 3


def test_library_has_no_driver_link_dependency():
    out = subprocess.run(["ldd", N.LIB_PATH], capture_output=True, text=True).stdout
    assert "libcuda.so" not in out and "libcudart" not in out and "libtorch" not in out


def test_compute_without_gpu_fails_loudly():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    with pytest.raises(MeaoError) as e:
        AmbientOcclusion(Camera(64, 64), device=0)
    assert e.value.code == N.MEAO_ERR_CUDA and "no CPU fallback" in str(e.value)
    plan = AmbientOcclusion(Camera(64, 64), device=-1)          # planning-only context
    with pytest.raises(MeaoError) as e2:
        plan.render_host(np.zeros((64, 64), np.float32))
    assert e2.value.code == N.MEAO_ERR_CUDA


def test_default_params_match_component():
    p = N.MeaoParams()
    N.lib().meao_default_params(C.byref(p))
    assert (p.noise_filter_tolerance, p.upsample_tolerance, p.thickness_modifier, p.intensity) == (0.0, -12.0, 1.0, 1.0)
    assert abs(p.blur_tolerance + 4.6) < 1e-6 and p.debug == 0 and p.ambient_only == 1     # AO.cs:20-68


@pytest.mark.parametrize("W,H", [(3840, 2160), (1920, 1080), (256, 256), (641, 363)])
@pytest.mark.parametrize("kw", [dict(), dict(intensity=1.1, thickness_modifier=3.0, blur_tolerance=-2.5, upsample_tolerance=-7.0, noise_filter_tolerance=-4.0)])
def test_planner_constants_equal_oracle_constants(W, H, kw):
    ao = AmbientOcclusion(Camera(W, H), device=-1)
    for py, cs in (("noise_filter_tolerance", "noiseFilterTolerance"), ("blur_tolerance", "blurTolerance"), ("upsample_tolerance", "upsampleTolerance"),
                   ("thickness_modifier", "thicknessModifier"), ("intensity", "intensity")):
        if py in kw:
            setattr(ao, cs, kw[py])
    o = Oracle(W, H, tan_half_fov_h_=1.0 / Camera(W, H).projection00, **kw)
    assert np.array_equal(ao.zbuffer_params(), o.zbuffer_params())
    for k in range(1, 5):
        a, b = ao.render_constants(k), o.render_constants(k)
        for key in a:
            assert np.array_equal(np.asarray(a[key]), np.asarray(b[key])), (k, key)
        a, b = ao.upsample_constants(k), o.upsample_constants(k)
        for key in a:
            assert np.array_equal(np.asarray(a[key]), np.asarray(b[key])), (k, key)


def test_late_update_change_detection():
    """CheckPropertiesChanged / CheckBaseDimensions semantics (AO.cs:104-113, 338-341)."""
    ao = AmbientOcclusion(Camera(640, 360), device=-1)
    assert ao.LateUpdate() is True          # first frame: size set
    assert ao.LateUpdate() is False
    ao.intensity = 1.5
    assert ao.LateUpdate() is True
    ao.intensity = 1.5
    assert ao.LateUpdate() is False
    ao.ambientOnly = False                  # not part of CheckPropertiesChanged in the reference either
    assert ao.LateUpdate() is False
    ao.camera.pixelWidth = 800
    assert ao.LateUpdate() is True
    assert ao.rebuild_count == 3


def test_algorithmic_bytes_match_survey_table():
    for (W, H), mb in (((256, 256), 1.040), ((1920, 1080), 32.908), ((3840, 2160), 131.614), ((7680, 4320), 526.439)):
        ao = AmbientOcclusion(Camera(W, H), device=-1)
        assert abs(ao.algorithmic_bytes(0) / 1e6 - mb) < 0.002
        assert ao.algorithmic_bytes(0) == sum(ao.algorithmic_bytes(s) for s in (1, 2, 3, 4))


def test_band_planning_halo_symmetry_and_limits():
    W, H = 7680, 4320
    bands = 8
    blocks = (H + 15) // 16
    cuts = [min(H, 16 * ((blocks * i) // bands)) for i in range(bands)] + [H]
    ctxs = []
    for i in range(bands):
        a = AmbientOcclusion(Camera(W, H), device=-1)
        a.set_row_band(cuts[i], cuts[i + 1], cuts[i - 1] if i > 0 else -1, cuts[i + 2] if i + 2 <= bands else -1)
        ctxs.append(a)
    for i in range(bands):
        rows = ctxs[i].band_rows()
        assert rows["produce"][0] == (cuts[i], cuts[i + 1])
        for k in range(1, 5):
            lo, hi = rows["need_low"][k]
            olo, ohi = rows["own_low"][k]
            assert lo <= olo and hi >= ohi
            assert olo == cuts[i] >> k
        for side, j in ((0, i - 1), (1, i + 1)):
            if 0 <= j < bands:
                assert ctxs[i].halo_rows(side, True) == ctxs[j].halo_rows(1 - side, False)      # what i sends == what j expects
                assert ctxs[i].halo_bytes(side) == ctxs[j].halo_recv_bytes(1 - side) > 0
            else:
                assert ctxs[i].halo_bytes(side) == 0
    # SURVEY.md 8(e): per-level halo is about 0.7 MB per direction at 8K, far below a raw-depth halo (346 rows)
    assert ctxs[3].halo_bytes(0) < 1.2e6
    thin = AmbientOcclusion(Camera(1920, 1088), device=-1)
    with pytest.raises(MeaoError) as e:
        thin.set_row_band(272, 544, 0, 816)
    assert e.value.code == N.MEAO_ERR_UNSUPPORTED
    with pytest.raises(MeaoError):
        thin.set_row_band(100, 544, 0, 816)         # not 16-row aligned


def test_pure_c_client_plans_without_gpu(tmp_path):
    """include/meao.h compiles as C99 and links against libmeao.so; the planner works and compute fails loudly."""
    exe = harness.build_c_client(tmp_path)
    r = subprocess.run([exe, "plan"], capture_output=True, text=True)
    assert r.returncode == 0 and "plan ok" in r.stdout, r.stderr


# ---- variants (SURVEY.md 8f.2 / 8f.4): planner side, no GPU ------------------------------------------------------
@pytest.mark.parametrize("W,H", [(3840, 2160), (641, 363)])
@pytest.mark.parametrize("exh,stereo", [(False, False), (True, False), (False, True), (True, True)])
def test_variant_constants_equal_oracle_constants(W, H, exh, stereo):
    cam = Camera(W // 2 if stereo else W, H, stereoEnabled=stereo)
    ao = AmbientOcclusion(cam, device=-1)
    ao.sampleExhaustively = exh
    ao.highQualityMask = 0b1010
    if stereo:
        ao.OnPreRender()                                         # one draw for both eyes => singlePassStereoEnabled (AO.cs:392-401)
    assert ao.LateUpdate() is True
    assert (ao._width, ao._height) == (2 * cam.pixelWidth if stereo else cam.pixelWidth, H)      # AO.cs:338-341
    # tanHalfFovH comes from the camera's own projection matrix (AO.cs:570-573), i.e. the single-eye aspect
    o = Oracle(ao._width, H, tan_half_fov_h_=1.0 / cam.projection00, sample_exhaustively=exh, single_pass_stereo=stereo, high_quality_mask=0b1010)
    for k in range(1, 5):
        for wide in (False, True):
            a, b = ao.render_constants(k, wide=wide), o.render_constants(k, wide=wide)
            for key in a:
                assert np.array_equal(np.asarray(a[key]), np.asarray(b[key])), (k, wide, key)
    assert ao.kernels_per_frame == 11
    v = N.MeaoVariants()
    N.check(ao._ctx, N.lib().meao_get_variants(ao._ctx, C.byref(v)))
    assert (v.single_pass_stereo, v.sample_exhaustively, v.high_quality_mask) == (int(stereo), int(exh), 0b1010)


def test_variant_change_detection_and_stereo_hack():
    """A variant change re-plans like a property change; the stereo detection keeps the reference's one-frame lag
    semantics (AO.cs:387-401: stereo is recognised only in a frame that saw exactly ONE OnPreRender)."""
    cam = Camera(640, 360, stereoEnabled=True)
    ao = AmbientOcclusion(cam, device=-1)
    assert ao.LateUpdate() is True and ao._width == 640        # no draw seen yet: not stereo (the first-frame glitch)
    ao.OnPreRender()
    assert ao.LateUpdate() is True and ao._width == 1280       # one draw for both eyes
    ao.OnPreRender(); ao.OnPreRender()
    assert ao.LateUpdate() is True and ao._width == 640        # multi-pass stereo: two draws
    ao.OnPreRender()
    cam.targetTexture = object()
    assert ao.LateUpdate() is False and ao._width == 640       # rendering to a texture: never single-pass (AO.cs:398)
    cam.targetTexture = None
    ao.sampleExhaustively = True
    assert ao.LateUpdate() is True
    assert ao.LateUpdate() is False
    ao.highQualityMask = 15
    assert ao.LateUpdate() is True and ao.kernels_per_frame == 13
    ao.highQualityMask = 16
    with pytest.raises(MeaoError):
        ao.LateUpdate()


def test_event_and_composite_pass_selection():
    """RegisterCommandBuffers / ambientOnlyEnabled (AO.cs:403-429): which camera events and which composite pass."""
    ao = AmbientOcclusion(Camera(64, 64), device=-1)
    assert ao.ambientOnlyEnabled is False and ao.camera_events == ("BeforeImageEffects", "BeforeImageEffects")
    ao.camera.actualRenderingPath = "DeferredShading"
    assert ao.ambientOnlyEnabled is True and ao.camera_events == ("BeforeReflections", "BeforeLighting")
    ao.camera.allowHDR = False
    assert ao.ambientOnlyEnabled is False
    ao.camera.allowHDR = True
    ao.ambientOnly = False
    assert ao.ambientOnlyEnabled is False
    ao.ambientOnly = True
    ao._debug = 6
    assert ao.camera_events == ("BeforeReflections", "AfterImageEffects")
    with pytest.raises(ValueError):
        ao.composite(None, color=None)


def test_csharp_host_binds_only_declared_entry_points():
    """host/AmbientOcclusionNative.cs cannot be compiled here (no C# toolchain): at least keep its P/Invoke surface in
    step with include/meao.h -- every extern it declares must be a declared + exported symbol, with the right arity."""
    cs = open(os.path.join(ROOT, "host", "AmbientOcclusionNative.cs")).read()
    externs = re.findall(r"static extern\s+\w+\s+(meao_[a-z0-9_]+)\s*\(([^)]*)\)", cs)
    assert len(externs) >= 12
    decl = set(_declared_functions())
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "meao.h")).read(), flags=re.S)
    for name, args in externs:
        assert name in decl, f"{name} is bound by the C# host but not declared in include/meao.h"
        m = re.search(r"\b" + name + r"\s*\(([^)]*)\)", hdr)
        n_c = 0 if m.group(1).strip() in ("", "void") else m.group(1).count(",") + 1
        n_cs = 0 if not args.strip() else args.count(",") + 1
        assert n_c == n_cs, f"{name}: {n_cs} parameters in C#, {n_c} in meao.h"
    # struct mirrors: field counts of the [StructLayout(Sequential)] twins
    for struct, n in (("MeaoParams", 7), ("MeaoCamera", 4), ("MeaoDeviceCfg", 2), ("MeaoVariants", 4)):
        body = re.search(r"public struct " + struct + r"\s*\{(.*?)\}", cs, flags=re.S).group(1)
        fields = sum(len(d.split(",")) for d in re.findall(r"public\s+(?:float|int|uint)\s+([^;]+);", body))
        assert fields == n, (struct, fields)


def test_csharp_scalar_twin_names_every_oracle_stage():
    """host/AmbientOcclusionScalar.cs is the (uncompilable here) C# twin of oracle/meao_oracle.c: it must cover the
    same stage functions and cite them."""
    cs = open(os.path.join(ROOT, "host", "AmbientOcclusionScalar.cs")).read()
    for fn in ("meao_oracle_create", "meao_oracle_downsample", "meao_oracle_render", "meao_oracle_upsample", "meao_oracle_run",
               "meao_oracle_f32_to_f16_bits", "meao_oracle_f16_bits_to_f32"):
        assert fn in cs, fn
    for method in ("Downsample", "Render", "Upsample", "Run", "TimeFrames", "Unorm8Code", "SampleThickness"):
        assert re.search(r"\b" + method + r"\s*\(", cs), method
    assert "(GI & 9) == 0" in cs            # Downsample1.compute:73 uses the OCTAL literal 011
    assert re.search(r"singleScale\s*&&\s*lo\s*==\s*1", cs)      # BASELINE configs[0]: the oracle's single_scale rule (Occlusion1 as LoResAO1)


# ---- round 2: ABI 3 -----------------------------------------------------------------------------------------------------------
def test_single_scale_variant_is_a_plan_input():
    ao = AmbientOcclusion(Camera(640, 360), device=-1)
    ao.LateUpdate()
    assert ao.kernels_per_frame == 9
    ao.singleScale = True
    assert ao.LateUpdate() is True and ao.kernels_per_frame == 3
    assert ao.LateUpdate() is False
    v = N.MeaoVariants()
    N.lib().meao_get_variants(ao._ctx, C.byref(v))
    assert v.single_scale == 1
    bad = N.MeaoVariants(0, 0, 3, 1)                     # single_scale excludes the high-quality passes
    assert N.lib().meao_set_variants(ao._ctx, C.byref(bad)) == N.MEAO_ERR_INVALID


def test_refused_row_band_leaves_the_context_untouched():
    """ADVICE r1: meao_set_row_band used to commit the band before validating the halo depth."""
    a = AmbientOcclusion(Camera(1920, 1088), device=-1)
    a.set_row_band(0, 544, -1, 1088)
    before = a.band_rows()
    with pytest.raises(MeaoError) as e:
        a.set_row_band(272, 544, 0, 816)                 # too thin for the level-4 halo
    assert e.value.code == N.MEAO_ERR_UNSUPPORTED
    assert a.band_rows() == before and a._band == (0, 544)
    assert a.halo_bytes(1) > 0 and a.halo_bytes(0) == 0


def test_resize_resets_band_in_the_host_mirror():
    cam = Camera(640, 720)
    a = AmbientOcclusion(cam, device=-1)
    a.set_row_band(0, 368, -1, 720)
    assert a._band_rows() == 368
    cam.pixelHeight = 360
    a.LateUpdate()
    assert a._band is None and a._band_rows() == 360 and a.band_rows()["produce"][0] == (0, 360)


def test_native_exchange_entry_points_need_a_device():
    a = AmbientOcclusion(Camera(640, 720), device=-1)
    a.set_row_band(0, 368, -1, 720)
    with pytest.raises(MeaoError) as e:
        a.band_export()
    assert e.value.code == N.MEAO_ERR_CUDA
    h = N.MeaoPeerHandle()
    assert N.lib().meao_band_connect(a._ctx, 1, C.byref(h)) == N.MEAO_ERR_CUDA
    assert N.lib().meao_band_step(a._ctx, None, 0, None, None) == N.MEAO_ERR_CUDA
    st = (C.c_int32 * 4)()
    assert N.lib().meao_band_status(a._ctx, st) == N.MEAO_ERR_INVALID
    assert C.sizeof(N.MeaoPeerHandle) == N.MEAO_PEER_HANDLE_BYTES == 128
    assert a.pdl_level == -1


def test_bad_depth_kind_is_refused_by_every_entry_point():
    """ADVICE r1: only meao_render validated depth_kind; the check now sits in the downsample recorder (shared by all entry
    points).  Without a device the calls fail earlier with MEAO_ERR_CUDA, so this checks the declared contract in the header."""
    hdr = open(os.path.join(ROOT, "include", "meao.h")).read()
    assert "MEAO_DEPTH_RAW_D24S8 = 3" in hdr
    src = open(os.path.join(ROOT, "miniengineao_b200", "csrc", "meao_api.cu")).read()
    rec = src[src.index("int record_downsample("):]
    assert "bad depth kind" in rec[:600]
