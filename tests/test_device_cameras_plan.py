"""CPU tests of device cameras (meao_bind_device_cameras) on plan-only contexts, which record the binding and allocate nothing: the return
values and refusals of bind and unbind, and that a refusal changes nothing; the frame generation, which moves on binding changes and not
on host camera changes while bound, except a reversed_z flip; meao_kernels_per_frame one higher while bound; the capacity against the
layer counts of a reservation; the row-band exclusion in both orders; and the Python component's deviceCameras property."""
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


def _bind(h, ptr, capacity):
    return N.lib().meao_bind_device_cameras(h, C.c_void_p(ptr) if ptr else None, capacity)


def _gen(h):
    return N.lib().meao_frame_generation(h)


def _error(h):
    return N.lib().meao_last_error(h).decode()


def _status(h):
    out = (C.c_int32 * 4)()
    rc = N.lib().meao_device_camera_status(h, out)
    return rc, list(out)


def _frame_rc(h):
    """meao_render on a plan-only context: MEAO_ERR_INVALID when refused before anything else, MEAO_ERR_CUDA when it got as far as the
    device (a plan-only context has none)."""
    return N.lib().meao_render(h, C.c_void_p(BUF2), N.MEAO_DEPTH_RAW_F32, C.c_void_p(BUF2 + 0x100000), None)


def test_bind_and_unbind():
    lib = N.lib()
    assert lib.meao_bind_device_cameras(None, None, 0) == N.MEAO_ERR_INVALID
    h = _create(3)
    assert _bind(h, 0, 0) == 0                              # nothing to unbind
    assert _status(h)[0] == N.MEAO_ERR_INVALID              # nothing bound
    g = _gen(h)
    assert _bind(h, BUF, 3) == 1 and _gen(h) == g + 1
    assert _bind(h, BUF, 3) == 0 and _gen(h) == g + 1       # the same binding
    assert _status(h) == (0, [0, 0, 0, 0])                  # plan-only: no status words
    assert _bind(h, BUF, 4) == 1 and _gen(h) == g + 2       # a new capacity
    assert _bind(h, BUF2, 4) == 1 and _gen(h) == g + 3      # a new pointer
    # refusals change nothing
    for ptr, cap, what in ((0, 3, "NULL"), (BUF, 0, "capacity 0"), (BUF, -1, "capacity -1"), (BUF, 65536, "capacity 65536"),
                           (BUF + 2, 3, "aligned")):
        assert _bind(h, ptr, cap) == N.MEAO_ERR_INVALID, (ptr, cap)
        assert what in _error(h), (what, _error(h))
        assert _gen(h) == g + 3
    assert _bind(h, BUF2, 4) == 0                           # still the binding it was
    assert _bind(h, BUF, 65535) == 1
    assert _bind(h, 0, 0) == 1 and _gen(h) == g + 5
    assert _bind(h, 0, 0) == 0
    lib.meao_destroy(h)


def test_kernels_per_frame_while_bound():
    lib = N.lib()
    for variants in ((0, 0, 0, 0), (1, 1, 15, 0), (0, 0, 0, 1)):
        h = _create(2)
        assert lib.meao_set_variants(h, C.byref(N.MeaoVariants(*variants))) >= 0
        n = lib.meao_kernels_per_frame(h)
        assert _bind(h, BUF, 2) == 1
        assert lib.meao_kernels_per_frame(h) == n + 1, variants
        assert _bind(h, 0, 0) == 1
        assert lib.meao_kernels_per_frame(h) == n
        lib.meao_destroy(h)


def test_host_camera_changes_while_bound():
    """A host camera change that keeps the Z direction is recorded only: no generation, and the getters describe the host cameras; a
    reversed_z flip stays structural; after the unbind the host cameras are those last set."""
    lib = N.lib()
    h = _create(2)
    assert _bind(h, BUF, 2) == 1
    g = _gen(h)
    assert lib.meao_set_camera(h, C.byref(N.MeaoCamera(0.25, 500.0, 1.5, 1))) == 0
    assert _gen(h) == g
    cams = (N.MeaoCamera * 2)(N.MeaoCamera(0.1, 90.0, 0.7, 1), N.MeaoCamera(2.0, 30.0, 3.0, 1))
    assert lib.meao_set_layer_cameras(h, cams, 2) == 1
    assert _gen(h) == g
    ref = _create(2, cam=(0.25, 500.0, 1.5, 1))
    assert lib.meao_set_layer_cameras(ref, cams, 2) == 1
    assert harness.plan_constants(h, 2) == harness.plan_constants(ref, 2)      # the getters keep describing the host cameras
    assert lib.meao_set_layer_cameras(h, None, 0) == 1 and _gen(h) == g
    assert lib.meao_set_layer_cameras(ref, None, 0) == 1
    assert harness.plan_constants(h, 2) == harness.plan_constants(ref, 2)
    # the Z direction is structural: it moves the generation whether or not a buffer is bound
    assert lib.meao_set_camera(h, C.byref(N.MeaoCamera(0.25, 500.0, 1.5, 0))) == 0
    assert _gen(h) == g + 1
    # projections stay structural too
    assert lib.meao_set_projection(h, N.MEAO_PROJECTION_ORTHOGRAPHIC) == 1 and _gen(h) == g + 2
    assert _bind(h, 0, 0) == 1
    assert lib.meao_set_projection(ref, N.MEAO_PROJECTION_ORTHOGRAPHIC) == 1
    assert lib.meao_set_camera(ref, C.byref(N.MeaoCamera(0.25, 500.0, 1.5, 0))) == 0
    assert harness.plan_constants(h, 2) == harness.plan_constants(ref, 2)
    lib.meao_destroy(h)
    lib.meao_destroy(ref)


def test_capacity_against_layer_counts_in_a_reservation():
    lib = N.lib()
    h = _create(2)
    assert lib.meao_reserve_layers(h, 8) == 1
    assert _bind(h, BUF, 4) == 1
    for L in (1, 3, 4, 5, 8, 2):
        lib.meao_set_layers(h, L)
        rc = _frame_rc(h)
        if L > 4:
            assert rc == N.MEAO_ERR_INVALID and "holds 4 cameras" in _error(h), (L, _error(h))
        else:
            assert rc == N.MEAO_ERR_CUDA, (L, rc, _error(h))        # past the capacity test: a plan-only context has no device
    # the stage calls are frames too
    lib.meao_set_layers(h, 6)
    assert lib.meao_stage_downsample(h, C.c_void_p(BUF2), N.MEAO_DEPTH_RAW_F32, None) == N.MEAO_ERR_INVALID
    assert "holds 4 cameras" in _error(h)
    # a capacity that covers the reservation serves every count
    assert _bind(h, BUF, 8) == 1
    for L in (8, 1, 5):
        lib.meao_set_layers(h, L)
        assert _frame_rc(h) == N.MEAO_ERR_CUDA
    lib.meao_destroy(h)


def test_row_bands_exclude_device_cameras_in_either_order():
    lib = N.lib()
    h = _create(1, W=128, H=256)
    assert lib.meao_set_row_band(h, 0, 128, -1, 256) == 0
    g = _gen(h)
    assert _bind(h, BUF, 1) == N.MEAO_ERR_UNSUPPORTED
    assert "row band" in _error(h) and _gen(h) == g
    assert _bind(h, 0, 0) == 0                              # nothing was bound
    lib.meao_destroy(h)

    h = _create(1, W=128, H=256)
    assert _bind(h, BUF, 1) == 1
    g = _gen(h)
    assert lib.meao_set_row_band(h, 0, 128, -1, 256) == N.MEAO_ERR_UNSUPPORTED
    assert "device camera" in _error(h) and _gen(h) == g
    rows = (C.c_int32 * 8)()
    assert lib.meao_halo_rows(h, 1, 1, rows) == N.MEAO_ERR_UNSUPPORTED
    assert lib.meao_halo_bytes(h, 1) == N.MEAO_ERR_UNSUPPORTED
    assert lib.meao_band_step(h, C.c_void_p(BUF2), N.MEAO_DEPTH_RAW_F32, C.c_void_p(BUF2), None) == N.MEAO_ERR_UNSUPPORTED
    out30 = (C.c_int32 * 30)()
    assert lib.meao_band_rows(h, out30) == 0 and out30[1] == 256     # still the whole frame
    assert _bind(h, 0, 0) == 1
    assert lib.meao_set_row_band(h, 0, 128, -1, 256) == 0
    lib.meao_destroy(h)


class _FakeCudaTensor:
    """What AmbientOcclusion.deviceCameras reads of a torch tensor, for a CPU-only test."""

    def __init__(self, n, ptr, dtype="torch.float32", contiguous=True):
        self.shape, self._ptr, self.dtype, self._contiguous, self.is_cuda = (n, 3), ptr, dtype, contiguous, True

    def dim(self):
        return 2

    def data_ptr(self):
        return self._ptr

    def is_contiguous(self):
        return self._contiguous


def test_python_device_cameras():
    lib = N.lib()
    cam = Camera(160, 90)
    ao = harness.context(cam)
    ao.layers = 2
    ao.LateUpdate()
    n = lib.meao_kernels_per_frame(ao._ctx)
    g = _gen(ao._ctx)
    t = _FakeCudaTensor(4, BUF)
    ao.deviceCameras = t
    assert ao.LateUpdate() is True
    assert lib.meao_kernels_per_frame(ao._ctx) == n + 1 and _gen(ao._ctx) == g + 1
    assert ao._boundCameraTensor is t                       # kept alive while bound
    assert ao.deviceCameraStatus() == (0, 0, 0)
    ao.LateUpdate()
    assert _gen(ao._ctx) == g + 1                           # the same data_ptr and n: no new binding
    ao.camera.nearClipPlane = 0.05                          # a host camera change while bound: no generation
    ao.LateUpdate()
    assert _gen(ao._ctx) == g + 1
    ao.deviceCameras = _FakeCudaTensor(4, BUF2)             # a new data_ptr binds again
    ao.LateUpdate()
    assert _gen(ao._ctx) == g + 2
    ao.deviceCameras = _FakeCudaTensor(3, BUF2)             # and a new length
    ao.LateUpdate()
    assert _gen(ao._ctx) == g + 3
    for bad in (_FakeCudaTensor(1, BUF), _FakeCudaTensor(4, BUF, dtype="torch.float64"), _FakeCudaTensor(4, BUF, contiguous=False)):
        ao.deviceCameras = bad
        with pytest.raises(ValueError, match="deviceCameras"):
            ao.LateUpdate()
    ao.deviceCameras = None
    ao.LateUpdate()
    assert lib.meao_kernels_per_frame(ao._ctx) == n and ao._boundCameraTensor is None
    with pytest.raises(N.MeaoError):
        ao.deviceCameraStatus()                             # nothing bound
    ao.close()
