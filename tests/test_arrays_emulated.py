"""CPU tests of CUDA-array frames (meao_render_arrays): the depth read from, the AO written into a 2-D, layered or cube-map CUDA array.

The array kernel sources (csrc/prepare_depth_array.cu, csrc/blur_upsample_array.cu) run in the fiber emulator with emulated arrays and
surface objects (tests/emu/frame_driver.cpp); every layer's AO, LinearDepth and LowDepth1..4 must be bit-identical to the oracle run on
that layer alone.  The emulated arrays have rows wider than the image with a marker in the spare bytes, and refuse any access that is
not one element at an element boundary, of the wrong shape, or out of range in trap mode.  Also here: the plan-only contract of the
three new entry points."""
import ctypes as C

import numpy as np
import pytest

from miniengineao_b200 import _native as N
from oracle.oracle import Oracle

from emu.emu import Frame  # noqa: E402  (tests/ is on sys.path via conftest)
from test_layers_emulated import _plan, _raw, contrasting_layers  # noqa: E402



def _d16(raw):
    codes = np.clip(np.rint(raw.astype(np.float64) * 65535), 0, 65535).astype(np.uint32)
    return codes.astype(np.uint16), (codes.astype(np.float32) * np.float32(1.0 / 65535)).astype(np.float32)


def _run_arrays(W, H, depth, *, depth_shape, ao_shape=None, linear=False, single_scale=False, oracle_depth=None, **kw):
    L = depth.shape[0]
    f = Frame(_plan(W, H, L, single_scale=single_scale, **kw), linear=linear)
    n0 = f.surface_accesses()
    ao = f.run_arrays(depth, depth_shape, ao_shape)
    assert f.surface_accesses() - n0 >= 2 * L * W * H          # every depth element loaded, every AO byte stored
    okw = dict(kw)
    if linear:
        okw["depth_is_linear"] = True
    if single_scale:
        okw["single_scale"] = True
    for l in range(L):
        orc = Oracle(W, H, threads=4, **okw)
        ref = orc.run(depth[l] if oracle_depth is None else oracle_depth[l])
        assert np.array_equal(ao[l], ref), (W, H, l, depth_shape, kw)
        for bid in (1, 2, 3, 4, 5):
            got = f.buffer(bid, l)
            want = orc.buffer(bid)
            if got.dtype == np.float16:
                with np.errstate(over="ignore"):
                    same = np.array_equal(got.view(np.uint16), want.astype(np.float16).view(np.uint16))
            else:
                same = np.array_equal(got.view(np.uint32), want.view(np.uint32))
            assert same, (W, H, l, bid, depth_shape, kw)
    return ao


@pytest.mark.parametrize("W,H", [(1, 1), (7, 5), (161, 93), (37, 70)])
def test_2d_arrays_ragged_sizes(W, H):
    """Widths that are not multiples of 8: the partial row ends take the per-element guards of both kernels."""
    _run_arrays(W, H, _raw(contrasting_layers(W, H, 1, seed=W)), depth_shape="2d", intensity=1.1)


@pytest.mark.parametrize("kind", ["raw_f32", "raw_f32_forward_z", "linear_f32", "d16", "d16_forward_z"])
def test_depth_kinds_three_layers(kind):
    W, H = 130, 70
    rz = "forward" not in kind
    lin = contrasting_layers(W, H, 3, seed=5)
    if kind == "linear_f32":
        _run_arrays(W, H, lin, depth_shape="layered", linear=True)
        return
    raw = _raw(lin, reversed_z=rz)
    if kind.startswith("d16"):
        codes, as_float = _d16(raw)
        _run_arrays(W, H, codes, depth_shape="layered", oracle_depth=as_float, reversed_z=rz)
    else:
        _run_arrays(W, H, raw, depth_shape="layered", reversed_z=rz)


@pytest.mark.parametrize("kw", [dict(high_quality_mask=1), dict(high_quality_mask=15), dict(single_scale=True),
                                dict(sample_exhaustively=True, reversed_z=False)])
def test_variants(kw):
    """high_quality_mask bit 0 selects the premin final level; single_scale feeds the final-style kernel with Occlusion1."""
    W, H = 150, 83
    depth = _raw(contrasting_layers(W, H, 3, seed=9), reversed_z=kw.get("reversed_z", True))
    _run_arrays(W, H, depth, depth_shape="layered", intensity=1.2, **kw)


@pytest.mark.parametrize("W", [96, 50])
def test_cube_maps(W):
    """Six square faces in a cube-map array; the AO may go to an array of another shape with the same layer count."""
    depth = _raw(contrasting_layers(W, W, 6, seed=W))
    _run_arrays(W, W, depth, depth_shape="cube")
    _run_arrays(W, W, depth, depth_shape="cube", ao_shape="layered", high_quality_mask=1)


def test_mixed_2d_and_layered_of_one_layer():
    W, H = 67, 45
    depth = _raw(contrasting_layers(W, H, 1, seed=2))
    _run_arrays(W, H, depth, depth_shape="layered", ao_shape="2d")


def test_interior_tiles_take_the_tma_path():
    """Big enough for TMA-fed interior tiles in the final level: the array kernel keeps the layered tile loop's box loads."""
    W, H = 640, 360
    depth = _raw(contrasting_layers(W, H, 2, seed=3))
    f = Frame(_plan(W, H, 2))
    n0 = f.tma_box_loads()
    ao = f.run_arrays(depth, "layered")
    assert f.tma_box_loads() - n0 > 300
    for l in range(2):
        assert np.array_equal(ao[l], Oracle(W, H, threads=4).run(depth[l])), l


# ---- plan-only contract ------------------------------------------------------------------------------------------------------
def test_array_entry_points_on_a_plan_only_context():
    from miniengineao_b200 import AmbientOcclusion, Camera
    lib = N.lib()
    a = AmbientOcclusion(Camera(64, 48), device=-1)
    a.LateUpdate()
    ctx = a._ctx
    fake = C.c_void_p(0x1000)
    assert lib.meao_render_arrays(ctx, fake, 0, fake, None) == N.MEAO_ERR_CUDA
    assert b"plan-only" in lib.meao_last_error(ctx)
    assert lib.meao_bind_event_arrays(ctx, 7, fake, 0, fake, None) == N.MEAO_ERR_CUDA
    assert lib.meao_release_array(ctx, fake) == N.MEAO_ERR_CUDA
    assert lib.meao_bind_event_arrays(ctx, 7, None, 0, None, None) == N.MEAO_OK       # unbinding needs no device
    for rc in (lib.meao_render_arrays(None, fake, 0, fake, None), lib.meao_bind_event_arrays(None, 7, fake, 0, fake, None),
               lib.meao_release_array(None, fake)):
        assert rc == N.MEAO_ERR_INVALID
    with pytest.raises(ValueError):
        a.render_arrays(1, 2, kind="d24")
