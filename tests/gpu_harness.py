"""Shared GPU helpers of the test suite: the torch and CUDA-runtime fixtures, CUDA arrays through ctypes, the half-second backlog the
no-wait tests put in front of their frames, connected row-band contexts on one device and a fresh context's frame.  Test modules
import the fixtures from here (`from gpu_harness import rt, torch_cuda`).  Nothing in it is collected by pytest."""
import ctypes as C

import numpy as np
import pytest

import harness

LAYERED, SURFACE_LOAD_STORE, CUBEMAP = 0x01, 0x02, 0x04
KIND_UNSIGNED, KIND_FLOAT, KIND_UNORM8, KIND_UNORM16 = 1, 2, 5, 8
H2D, D2H = 1, 2
SLEEP_CYCLES = 1 << 30          # about half a second of one spinning thread at the H100's clock: a backlog the host cannot outrun


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("GPU tests need a GPU")
    torch.cuda.init()
    return torch


@pytest.fixture(scope="module")
def rt(torch_cuda):
    return runtime()


# ---- CUDA arrays --------------------------------------------------------------------------------------------------------------------
class ChannelDesc(C.Structure):
    _fields_ = [("x", C.c_int), ("y", C.c_int), ("z", C.c_int), ("w", C.c_int), ("f", C.c_int)]


class Extent(C.Structure):
    _fields_ = [("width", C.c_size_t), ("height", C.c_size_t), ("depth", C.c_size_t)]


class Pos(C.Structure):
    _fields_ = [("x", C.c_size_t), ("y", C.c_size_t), ("z", C.c_size_t)]


class PitchedPtr(C.Structure):
    _fields_ = [("ptr", C.c_void_p), ("pitch", C.c_size_t), ("xsize", C.c_size_t), ("ysize", C.c_size_t)]


class Memcpy3DParms(C.Structure):
    _fields_ = [("srcArray", C.c_void_p), ("srcPos", Pos), ("srcPtr", PitchedPtr), ("dstArray", C.c_void_p), ("dstPos", Pos),
                ("dstPtr", PitchedPtr), ("extent", Extent), ("kind", C.c_int)]


def runtime():
    """The CUDA runtime (libcudart.so.12, loaded after torch so the process has one dynamic runtime) with the array calls typed."""
    r = C.CDLL("libcudart.so.12")
    r.cudaMallocArray.argtypes = [C.POINTER(C.c_void_p), C.POINTER(ChannelDesc), C.c_size_t, C.c_size_t, C.c_uint]
    r.cudaMalloc3DArray.argtypes = [C.POINTER(C.c_void_p), C.POINTER(ChannelDesc), Extent, C.c_uint]
    r.cudaFreeArray.argtypes = [C.c_void_p]
    r.cudaMemcpy3D.argtypes = [C.POINTER(Memcpy3DParms)]
    r.cudaMemcpy2DToArray.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_int]
    r.cudaMemcpy2DFromArray.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_int]
    return r


class Array:
    """A W x H CUDA array of `layers` layers: shape "2d" (layers 1), "layered" or "cube" (6), one channel of dtype."""
    DT = {np.dtype(np.float32): (32, KIND_FLOAT), np.dtype(np.uint16): (16, KIND_UNSIGNED), np.dtype(np.uint8): (8, KIND_UNSIGNED)}

    def __init__(self, rt, W, H, dtype, shape="2d", layers=1, flags=SURFACE_LOAD_STORE, kind=None, extra_flags=0):
        self.rt, self.W, self.H, self.dtype, self.shape = rt, W, H, np.dtype(dtype), shape
        self.layers = 6 if shape == "cube" else layers
        bits, k = self.DT[self.dtype]
        desc = ChannelDesc(bits, 0, 0, 0, k if kind is None else kind)
        h = C.c_void_p()
        if shape == "2d":
            rc = rt.cudaMallocArray(C.byref(h), C.byref(desc), W, H, flags | extra_flags)
        else:
            f = flags | extra_flags | (CUBEMAP if shape == "cube" else LAYERED)
            rc = rt.cudaMalloc3DArray(C.byref(h), C.byref(desc), Extent(W, H, self.layers), f)
        assert rc == 0, f"array allocation failed ({rc})"
        self.handle = h.value

    def _copy(self, host, to_array):
        if self.shape == "2d":
            wb = self.W * self.dtype.itemsize
            if to_array:
                rc = self.rt.cudaMemcpy2DToArray(C.c_void_p(self.handle), 0, 0, C.c_void_p(host.ctypes.data), wb, wb, self.H, H2D)
            else:
                rc = self.rt.cudaMemcpy2DFromArray(C.c_void_p(host.ctypes.data), wb, C.c_void_p(self.handle), 0, 0, wb, self.H, D2H)
        else:
            p = Memcpy3DParms()
            hp = PitchedPtr(host.ctypes.data, self.W * self.dtype.itemsize, self.W, self.H)
            if to_array:
                p.srcPtr, p.dstArray, p.kind = hp, self.handle, H2D
            else:
                p.srcArray, p.dstPtr, p.kind = self.handle, hp, D2H
            p.extent = Extent(self.W, self.H, self.layers)
            rc = self.rt.cudaMemcpy3D(C.byref(p))
        assert rc == 0, f"array copy failed ({rc})"

    def fill(self, img):
        self._copy(np.ascontiguousarray(img.reshape(self.layers, self.H, self.W), dtype=self.dtype), True)

    def read(self):
        out = np.empty((self.layers, self.H, self.W), self.dtype)
        self._copy(out, False)
        return out

    def free(self):
        if self.handle:
            assert self.rt.cudaFreeArray(C.c_void_p(self.handle)) == 0
            self.handle = None


# ---- frames ---------------------------------------------------------------------------------------------------------------------
def backlog(torch, s, ao, d, out, n=50):
    """A spinning kernel, then n frames at the current size into `out`, then an event E, all on stream s: E completes half a second
    from now."""
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP_CYCLES)
    for _ in range(n):
        ao.render(d, out, stream=s)
    e = torch.cuda.Event()
    e.record(s)
    return e


def fresh_frame(torch, ao, depth):
    """The AO and every debug buffer of the first frame of the new context `ao` on `depth`; closes `ao`."""
    out = ao.render(torch.from_numpy(np.ascontiguousarray(depth)).cuda()).cpu().numpy()
    bufs = {bid: ao.debug_buffer(bid) for bid in harness.buffer_ids()}
    ao.close()
    return out, bufs


def native_bands(torch, W, H, bands, device=0, **attrs):
    """`bands` band contexts on ONE device, connected to each other through meao_band_export / meao_band_connect (in-process:
    direct pointers) -- the same kernels, flags and graph as across GPUs, minus NVLink.  attrs: AmbientOcclusion properties."""
    from miniengineao_b200 import rowtile
    cuts = rowtile.partition(H, bands)
    ctxs = []
    for i in range(bands):
        a = harness.context(W, H, device=device)
        for k, v in attrs.items():
            setattr(a, k, v)
        a.set_row_band(cuts[i], cuts[i + 1], *rowtile.neighbours(cuts, i))
        ctxs.append(a)
    handles = [a.band_export() for a in ctxs]
    for i, a in enumerate(ctxs):
        if i > 0:
            a.band_connect(0, handles[i - 1])
        if i + 1 < bands:
            a.band_connect(1, handles[i + 1])
    streams = [torch.cuda.Stream() for _ in range(bands)]      # one stream per band, like one GPU per band: the exchange kernels must overlap
    return cuts, ctxs, streams
