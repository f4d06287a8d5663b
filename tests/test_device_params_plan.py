"""CPU tests of device parameters (meao_bind_device_params) on plan-only contexts, which record the binding and allocate nothing: the
return values and refusals of bind and unbind, and that a refusal changes nothing; the frame generation, which moves on binding changes and
not on host thickness_modifier / intensity changes while bound, while a tolerance change still moves it; the constant getters, which keep
describing the host values; meao_kernels_per_frame one higher while bound, with and without device cameras at every hierarchy depth; the
row-band exclusion in both orders; the profile name of the stage; and the Python component's deviceParams property."""
import ctypes as C

import pytest

import harness
from miniengineao_b200 import Camera
from miniengineao_b200 import _native as N

CAM = (0.5, 80.0, 6.0, 1)
BUF = 0x7f0000001000         # a plan-only context never dereferences the buffer
BUF2 = 0x7f0000002000


def _create(layers=1, W=160, H=96, cam=CAM):
    lib = N.lib()
    h = C.c_void_p()
    assert lib.meao_create(C.byref(N.MeaoDeviceCfg(-1, 0)), C.byref(h)) == 0
    assert lib.meao_set_camera(h, C.byref(N.MeaoCamera(*cam))) == 0
    if layers != 1:
        assert lib.meao_set_layers(h, layers) == 1
    if W:
        assert lib.meao_resize(h, W, H) == 1
    return h


def _bind(h, ptr):
    return N.lib().meao_bind_device_params(h, C.c_void_p(ptr) if ptr else None)


def _gen(h):
    return N.lib().meao_frame_generation(h)


def _error(h):
    return N.lib().meao_last_error(h).decode()


def _status(h):
    out = (C.c_int32 * 4)()
    rc = N.lib().meao_device_param_status(h, out)
    return rc, list(out)


def _params(h, **kw):
    p = N.MeaoParams()
    N.lib().meao_get_params(h, C.byref(p))
    for k, v in kw.items():
        setattr(p, k, v)
    return N.lib().meao_set_params(h, C.byref(p))


def test_bind_and_unbind():
    lib = N.lib()
    assert lib.meao_bind_device_params(None, None) == N.MEAO_ERR_INVALID
    assert lib.meao_device_param_status(None, (C.c_int32 * 4)()) == N.MEAO_ERR_INVALID
    h = _create(3)
    assert _bind(h, 0) == 0                                 # nothing to unbind
    assert _status(h)[0] == N.MEAO_ERR_INVALID              # nothing bound
    g = _gen(h)
    assert _bind(h, BUF) == 1 and _gen(h) == g + 1
    assert _bind(h, BUF) == 0 and _gen(h) == g + 1          # the same pointer
    assert _status(h) == (0, [0, 0, 0, 0])                  # plan-only: no status words
    assert _bind(h, BUF2) == 1 and _gen(h) == g + 2         # a new pointer
    for ptr in (BUF + 2, BUF + 1, BUF2 + 3):                # not 4-byte aligned: refused, nothing changes
        assert _bind(h, ptr) == N.MEAO_ERR_INVALID, ptr
        assert "aligned" in _error(h) and _gen(h) == g + 2
    assert _bind(h, BUF2) == 0                              # still the binding it was
    assert _bind(h, 0) == 1 and _gen(h) == g + 3
    assert _bind(h, 0) == 0 and _gen(h) == g + 3
    assert _status(h)[0] == N.MEAO_ERR_INVALID
    lib.meao_destroy(h)


@pytest.mark.parametrize("cams", [False, True])
def test_kernels_per_frame_while_bound(cams):
    lib = N.lib()
    for depth in (1, 2, 3, 4):
        for variants in ((0, 0, 0, 0), (1, 1, 15, 0), (0, 0, 5, 0)):
            h = _create(2)
            assert lib.meao_set_variants(h, C.byref(N.MeaoVariants(*variants))) >= 0
            assert lib.meao_set_hierarchy_depth(h, depth) >= 0
            if cams:
                assert lib.meao_bind_device_cameras(h, C.c_void_p(BUF2), 2) == 1
            hq = sum(1 for k in range(depth) if (variants[2] >> k) & 1)
            n = 1 + 2 * depth + hq + (1 if cams else 0)
            assert lib.meao_kernels_per_frame(h) == n, (depth, variants)
            assert _bind(h, BUF) == 1
            assert lib.meao_kernels_per_frame(h) == n + 1, (depth, variants)
            assert _bind(h, 0) == 1
            assert lib.meao_kernels_per_frame(h) == n
            lib.meao_destroy(h)


def test_host_parameter_changes_while_bound():
    """A change of thickness_modifier / intensity alone is recorded only: it returns 1, moves no generation, and the getters describe the
    host values; a tolerance change behaves as without a binding; after the unbind the host values are those last set."""
    lib = N.lib()
    h, ref = _create(2), _create(2)
    assert _bind(h, BUF) == 1
    g = _gen(h)
    assert _params(h, thickness_modifier=2.5) == 1 and _gen(h) == g
    assert _params(h, intensity=0.25) == 1 and _gen(h) == g
    assert _params(h, thickness_modifier=0.75, intensity=1.5) == 1 and _gen(h) == g
    assert _params(h, thickness_modifier=0.75, intensity=1.5) == 0 and _gen(h) == g       # the same values
    assert _params(ref, thickness_modifier=0.75, intensity=1.5) == 1
    assert harness.plan_constants(h, 2) == harness.plan_constants(ref, 2)      # the getters keep describing the host values
    # refusals stay refusals
    assert _params(h, thickness_modifier=0.0) == N.MEAO_ERR_INVALID and _gen(h) == g
    # the tolerances stay host frame constants; so does debug
    assert _params(h, upsample_tolerance=-10.0) == 1 and _gen(h) == g + 1
    assert _params(h, blur_tolerance=-4.0, intensity=0.5) == 1 and _gen(h) == g + 2
    assert _params(h, debug=1) == 1 and _gen(h) == g + 3
    assert _params(ref, upsample_tolerance=-10.0, blur_tolerance=-4.0, intensity=0.5, debug=1) == 1
    assert harness.plan_constants(h, 2) == harness.plan_constants(ref, 2)
    assert _params(h, thickness_modifier=3.0) == 1 and _gen(h) == g + 3
    assert _bind(h, 0) == 1 and _gen(h) == g + 4
    assert _params(h, intensity=0.5) == 0 and _gen(h) == g + 4                 # unbound: the host values are those last set
    assert _params(h, intensity=0.6) == 1 and _gen(h) == g + 5                 # and a change moves the generation again
    assert _params(ref, thickness_modifier=3.0, intensity=0.6) == 1
    assert harness.plan_constants(h, 2) == harness.plan_constants(ref, 2)
    lib.meao_destroy(h)
    lib.meao_destroy(ref)


def test_getters_after_a_size_switch_while_bound():
    """A parked size keeps its older plan: after a host change while bound it plans the host values again before the getters answer."""
    lib = N.lib()
    h, ref = _create(1), _create(1)
    assert lib.meao_reserve(h, 320, 192) >= 0
    assert _bind(h, BUF) == 1
    assert lib.meao_resize(h, 320, 192) == 1
    assert _params(h, intensity=0.4, thickness_modifier=4.0) == 1
    assert lib.meao_resize(h, 160, 96) == 1
    assert _params(ref, intensity=0.4, thickness_modifier=4.0) == 1
    assert harness.plan_constants(h, 1) == harness.plan_constants(ref, 1)
    lib.meao_destroy(h)
    lib.meao_destroy(ref)


def test_row_bands_exclude_device_params_in_either_order():
    lib = N.lib()
    h = _create(1, W=128, H=256)
    assert lib.meao_set_row_band(h, 0, 128, -1, 256) == 0
    g = _gen(h)
    assert _bind(h, BUF) == N.MEAO_ERR_UNSUPPORTED
    assert "row band" in _error(h) and _gen(h) == g
    assert _bind(h, 0) == 0                                 # nothing was bound
    lib.meao_destroy(h)

    h = _create(1, W=128, H=256)
    assert _bind(h, BUF) == 1
    g = _gen(h)
    assert lib.meao_set_row_band(h, 0, 128, -1, 256) == N.MEAO_ERR_UNSUPPORTED
    assert "device parameter" in _error(h) and _gen(h) == g
    rows = (C.c_int32 * 8)()
    assert lib.meao_halo_rows(h, 1, 1, rows) == N.MEAO_ERR_UNSUPPORTED
    assert lib.meao_halo_bytes(h, 1) == N.MEAO_ERR_UNSUPPORTED
    assert lib.meao_band_step(h, C.c_void_p(BUF2), N.MEAO_DEPTH_RAW_F32, C.c_void_p(BUF2), None) == N.MEAO_ERR_UNSUPPORTED
    assert "device parameter" in _error(h) and _gen(h) == g
    out30 = (C.c_int32 * 30)()
    assert lib.meao_band_rows(h, out30) == 0 and out30[1] == 256     # still the whole frame
    assert _bind(h, 0) == 1
    assert lib.meao_set_row_band(h, 0, 128, -1, 256) == 0
    lib.meao_destroy(h)


class _FakeCudaTensor:
    """What AmbientOcclusion.deviceParams reads of a torch tensor, for a CPU-only test."""

    def __init__(self, ptr, shape=(2,), dtype="torch.float32", contiguous=True):
        self.shape, self._ptr, self.dtype, self._contiguous, self.is_cuda = shape, ptr, dtype, contiguous, True

    def dim(self):
        return len(self.shape)

    def data_ptr(self):
        return self._ptr

    def is_contiguous(self):
        return self._contiguous


def test_python_device_params():
    lib = N.lib()
    cam = Camera(160, 90)
    ao = harness.context(cam)
    ao.layers = 2
    ao.LateUpdate()
    n = lib.meao_kernels_per_frame(ao._ctx)
    g = _gen(ao._ctx)
    t = _FakeCudaTensor(BUF)
    ao.deviceParams = t
    assert ao.LateUpdate() is True
    assert lib.meao_kernels_per_frame(ao._ctx) == n + 1 and _gen(ao._ctx) == g + 1
    assert ao._boundParamTensor is t                        # kept alive while bound
    assert ao.deviceParamStatus() == (0, 0)
    ao.LateUpdate()
    assert _gen(ao._ctx) == g + 1                           # the same data_ptr: no new binding
    ao.intensity = 0.3                                      # a host intensity change while bound: no generation
    ao.thicknessModifier = 2.0
    ao.LateUpdate()
    assert _gen(ao._ctx) == g + 1
    ao.deviceParams = _FakeCudaTensor(BUF2)                 # a new data_ptr binds again
    ao.LateUpdate()
    assert _gen(ao._ctx) == g + 2
    for bad in (_FakeCudaTensor(BUF, shape=(3,)), _FakeCudaTensor(BUF, shape=(1, 2)), _FakeCudaTensor(BUF, dtype="torch.float64"),
                _FakeCudaTensor(BUF, contiguous=False)):
        ao.deviceParams = bad
        with pytest.raises(ValueError, match="deviceParams"):
            ao.LateUpdate()
    ao.deviceParams = None
    ao.LateUpdate()
    assert lib.meao_kernels_per_frame(ao._ctx) == n and ao._boundParamTensor is None
    with pytest.raises(N.MeaoError):
        ao.deviceParamStatus()                              # nothing bound
    ao.close()
