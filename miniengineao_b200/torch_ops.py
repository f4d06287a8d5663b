"""The AO frame as torch.library operators, for torch.compile: `meao::ambient_occlusion` (one [H, W] or layered [L, H, W] depth) and
`meao::ambient_occlusion_batch` (a list of [H, W] depths, one layer each).  Dynamo traces either as one opaque node with known output
shapes, without a graph break, and the graph trees of torch.compile(mode="reduce-overhead") record the frame's kernels into their own
CUDA graph (include/meao.h, "frames inside a caller's graph").

The operators run on AmbientOcclusion instances: `render` / `render_batch` on torch's current stream of the depth's device, the depth
read in place through its strides (meao_render_pitched) and a new contiguous uint8 AO.  Nothing is copied or converted; the only other
device work is the copy of a `cameras` tensor into the context's bound camera buffer, and of a `render_params` tensor into its bound
parameter buffer.

Cameras, chosen by the caller's input:
  - `cameras`, a CUDA float32 tensor [L, 3] of (near_clip, far_clip, tan_half_fov_h) per layer: a camera that may move every call.  The
    context binds a buffer of its own once (meao_bind_device_cameras) and every call copies `cameras` into it on the stream, so a
    replayed graph follows new cameras without a re-capture.
  - `camera`, a list (near_clip, far_clip, tan_half_fov_h): a fixed host camera, part of the context key below.  It spares the frame the
    camera stage and the layered kernels that device cameras take at L = 1 (DESIGN.md 2.18).
Exactly one of the two is given.  tan_half_fov_h is 1 / projection[0, 0]: the half-width of the view volume under an orthographic
projection.

Contexts.  A frame recorded into a caller's graph replays the plan, constants and buffers it was recorded with, so a context must never
change once a frame of it may sit in such a graph.  Contexts are cached per process, keyed by everything a context is configured with:
the frame form, device, L, H, W, kind, the MeaoParams floats, reversed_z, the projection (or per-layer projection table), the
MeaoVariants fields, the hierarchy depth and the host camera.  A new value of any of these gets a new context, and no context is ever
handed a new value.  The parameters are floats of the operator's schema, which Dynamo specialises on: a new intensity is a new compiled
graph and a new context, not a per-frame knob.  Nothing is evicted; release_contexts() drops them all.

Thickness and intensity that change every call: `render_params`, a CUDA float32 tensor [2] of (thickness_modifier, intensity), the
operators' last argument.  The context binds a buffer of its own once (meao_bind_device_params) and every call copies `render_params`
into it on the stream, as for `cameras`, so a fade runs in one compiled graph and one context.  The key then holds "device" in place of
those two floats, and the schema floats thickness_modifier and intensity are ignored.

A context is created and settled by a frame issued outside any stream capture.  torch.cuda.graph's documented warm-up and the graph
trees' warm-up run every call eagerly first; a first call for a key inside a capture raises.  After its first frame each context's
meao_frame_generation is recorded and checked after every later frame, so a context that changed under a recorded frame raises.

No autograd: the AO is UNORM8 codes.  Import this module (or read miniengineao_b200.ambient_occlusion_op) before calling
torch.ops.meao.*: importing it registers the operators.
"""
import threading
from typing import List, Optional, Sequence, Union

import numpy as np
import torch

from . import _native as N
from .ambient_occlusion import AmbientOcclusion, Camera

PERSPECTIVE, ORTHOGRAPHIC = N.MEAO_PROJECTION_PERSPECTIVE, N.MEAO_PROJECTION_ORTHOGRAPHIC
_PROJECTION_NAMES = {"perspective": PERSPECTIVE, "orthographic": ORTHOGRAPHIC}
# depth dtypes per kind, AmbientOcclusion._kind's rule; d24s8: D24_UNORM_S8_UINT words, depth in the low 24 bits (MEAO_DEPTH_RAW_D24S8)
KIND_DTYPES = {"raw_f32": (torch.float32,), "linear_f32": (torch.float32,), "d16": (torch.uint16,), "d24s8": (torch.int32, torch.uint32)}
MAX_BATCH = 256             # MEAO_MAX_BATCH
MAX_LAYERS = 65535          # meao_set_layers, meao_bind_device_cameras
MAX_SIZE = 32768            # meao_resize


# ---- validation, shared by the fake and the real implementations ------------------------------------------------------------------
def _check_view(t: torch.Tensor, name: str) -> None:
    """A view the frame reads in place: last stride 1 and positive other strides (a dimension of size 1 is never stepped along)."""
    for i in range(t.dim()):
        if t.shape[i] > 1 and (t.stride(i) != 1 if i == t.dim() - 1 else t.stride(i) <= 0):
            raise ValueError(f"{name} must have a last-dimension stride of 1 and positive other strides (got strides {tuple(t.stride())}): "
                             "the operator reads the view in place and never copies it")


def _check_inputs(depths: Sequence[torch.Tensor], layers: int, cameras: Optional[torch.Tensor], camera: Optional[List[float]], kind: str,
                  projection: int, layer_projections: Optional[List[int]], single_pass_stereo: bool, high_quality_mask: int,
                  hierarchy_depth: int, batch: bool) -> None:
    """Every refusal that needs no context: device, dtype, rank, layer count, strides, the camera forms and the enum ranges."""
    if kind not in KIND_DTYPES:
        raise ValueError(f"kind must be one of {sorted(KIND_DTYPES)} (got {kind!r})")
    d0 = depths[0]
    for i, d in enumerate(depths):
        name = f"depths[{i}]" if batch else "depth"
        if d.device.type != "cuda":
            raise ValueError(f"{name} must be a CUDA tensor (got device {d.device})")
        if d.device != d0.device:
            raise ValueError(f"{name} is on {d.device}, depths[0] on {d0.device}")
        if d.dtype not in KIND_DTYPES[kind]:
            want = " or ".join(str(t).replace("torch.", "") for t in KIND_DTYPES[kind])
            raise ValueError(f"{name} of kind {kind!r} must be {want} (got {str(d.dtype).replace('torch.', '')})")
        if d.shape[-2:] != d0.shape[-2:]:
            raise ValueError(f"{name} is {tuple(d.shape)}, depths[0] {tuple(d0.shape)}: every layer has one size")
        _check_view(d, name)
    H, W = d0.shape[-2], d0.shape[-1]
    if not (1 <= H <= MAX_SIZE and 1 <= W <= MAX_SIZE):
        raise ValueError(f"depth is {W} x {H}: width and height must be in 1..{MAX_SIZE}")
    if not 1 <= layers <= (MAX_BATCH if batch else MAX_LAYERS):
        raise ValueError(f"{layers} layers: 1..{MAX_BATCH if batch else MAX_LAYERS} allowed")
    if single_pass_stereo and W % 2:
        raise ValueError(f"single_pass_stereo needs the double-wide eye pair: an even width (got {W})")
    if (cameras is None) == (camera is None):
        raise ValueError("pass exactly one of `cameras` (a CUDA float32 tensor [L, 3]) and `camera` (a list of 3 floats)")
    if cameras is not None:
        if cameras.device != d0.device or cameras.dtype != torch.float32 or cameras.dim() != 2 or cameras.shape[0] != layers \
                or cameras.shape[1] != 3:
            raise ValueError(f"cameras must be a float32 tensor [{layers}, 3] on {d0.device} (got {str(cameras.dtype).replace('torch.', '')} "
                             f"{tuple(cameras.shape)} on {cameras.device})")
    else:
        if len(camera) != 3:
            raise ValueError(f"camera must be (near_clip, far_clip, tan_half_fov_h) (got {len(camera)} values)")
        near, far, tan = camera
        if not (near > 0 and far > near and tan > 0):
            raise ValueError(f"camera {tuple(camera)}: near_clip > 0, far_clip > near_clip and tan_half_fov_h > 0 required")
    projections = [projection] + list(layer_projections or [])
    if any(p not in (PERSPECTIVE, ORTHOGRAPHIC) for p in projections):
        raise ValueError(f"projections must be {PERSPECTIVE} (perspective) or {ORTHOGRAPHIC} (orthographic) (got {projections})")
    if layer_projections is not None:
        if len(layer_projections) != layers:
            raise ValueError(f"layer_projections has {len(layer_projections)} entries for {layers} layers")
        if batch and ORTHOGRAPHIC in layer_projections:
            raise ValueError("a batch takes no per-layer table with an orthographic entry (meao_set_layer_projections); "
                             "use projection=ORTHOGRAPHIC for a batch of orthographic views")
    if not 0 <= high_quality_mask <= 15:
        raise ValueError(f"high_quality_mask must be in 0..15 (got {high_quality_mask})")
    if not 1 <= hierarchy_depth <= 4:
        raise ValueError(f"hierarchy_depth must be in 1..4 (got {hierarchy_depth})")


# ---- contexts ---------------------------------------------------------------------------------------------------------------------
def _f32(x: float) -> float:
    """The value the library stores (a C float): the key of 1.1 and of float32(1.1) is the same."""
    return float(np.float32(x))


def context_key(form: str, device: int, layers: int, height: int, width: int, kind: str, cameras_on_device: bool,
                camera: Optional[Sequence[float]], params: Sequence[float], reversed_z: bool, projection: int,
                layer_projections: Optional[Sequence[int]], variants: Sequence[int], hierarchy_depth: int,
                params_on_device: bool = False) -> tuple:
    """The cache key of a context: form ("frame" or "batch"), device ordinal, L, H, W, kind, the five MeaoParams floats, reversed_z, the
    projection and projection table, the MeaoVariants fields (single_pass_stereo, sample_exhaustively, high_quality_mask, single_scale),
    the hierarchy depth, and the host camera (None: cameras from the bound device buffer).  params_on_device: thickness_modifier and
    intensity come from the bound device parameter buffer, and the key holds "device" in place of those two floats."""
    params = tuple(_f32(p) for p in params)
    if params_on_device:
        params = params[:3] + ("device", "device")
    return (form, int(device), int(layers), int(height), int(width), kind, params, bool(reversed_z),
            int(projection), None if layer_projections is None else tuple(int(p) for p in layer_projections),
            tuple(int(v) for v in variants), int(hierarchy_depth),
            "device" if cameras_on_device else tuple(_f32(c) for c in camera))


class _HostCamera(Camera):
    """A Camera whose 1 / projection00 is the given tan_half_fov_h itself (for a float32 value, exactly), not one derived from a vertical
    field of view: the value a `cameras` row carries."""

    def __init__(self, width: int, height: int, near: float, far: float, tan_half_fov_h: float, reversed_z: bool, stereo: bool):
        super().__init__(width, height, nearClipPlane=near, farClipPlane=far, usesReversedZBuffer=reversed_z, stereoEnabled=stereo)
        self.tanHalfFovH = tan_half_fov_h

    @property
    def projection00(self) -> float:
        return 1.0 / self.tanHalfFovH


def _outside_graph_pools(alloc):
    """alloc() on a helper thread.  The graph trees of torch.compile route every allocation of the calling thread to their private pool
    while they warm up or record a function, and check that nothing but the function's outputs stays alive there; a context's camera
    buffer (or parameter buffer), made by the first call for its key (a warm-up), outlives every graph, so it comes from the ordinary
    pool."""
    out = []
    t = threading.Thread(target=lambda: out.append(alloc()))
    t.start()
    t.join()
    if not out:
        raise RuntimeError("meao: allocating a context's camera buffer failed")
    return out[0]


class _Context:
    """One AmbientOcclusion configured once from its key, its bound camera and parameter buffers and the generation recorded after its
    first frame."""

    def __init__(self, key: tuple):
        form, device, L, H, W, kind, params, reversed_z, projection, table, variants, depth, camera = key
        stereo, exhaustive, hq, single_scale = variants
        near, far, tan = (0.3, 100.0, 1.0) if camera == "device" else camera      # a valid host camera under device ones
        cam = _HostCamera(W // 2 if stereo else W, H, near, far, tan, reversed_z, bool(stereo))
        ao = AmbientOcclusion(cam, device=device)
        params_on_device = params[3] == "device"
        if params_on_device:
            params = params[:3] + (1.0, 1.0)        # valid host values under device ones
        (ao.noiseFilterTolerance, ao.blurTolerance, ao.upsampleTolerance, ao.thicknessModifier, ao.intensity) = params
        ao.sampleExhaustively, ao.highQualityMask, ao.singleScale, ao.hierarchyDepth = bool(exhaustive), hq, bool(single_scale), depth
        ao.layers = L
        if table is not None:
            # the per-layer projection table goes through layerCameras (AmbientOcclusion._layer_projections): every layer with the
            # context's host camera, each with its own projection
            ao.perLayerProjection = True
            ao.layerCameras = [_HostCamera(cam.pixelWidth, H, near, far, tan, reversed_z, bool(stereo)) for _ in table]
            for c, p in zip(ao.layerCameras, table):
                c.orthographic = p == ORTHOGRAPHIC
        cam.orthographic = projection == ORTHOGRAPHIC
        self.cameras = None
        if camera == "device" and device >= 0:
            self.cameras = _outside_graph_pools(lambda: torch.empty((L, 3), dtype=torch.float32, device=f"cuda:{device}"))
            ao.deviceCameras = self.cameras
        self.params = None
        if params_on_device and device >= 0:
            self.params = _outside_graph_pools(lambda: torch.tensor(params[3:], dtype=torch.float32, device=f"cuda:{device}"))
            ao.deviceParams = self.params
        self.key, self.ao, self.form, self.kind, self.stereo = key, ao, form, kind, bool(stereo)
        self.generation = None
        self._settle()

    def _settle(self) -> None:
        """Applies the configuration (a re-plan, outside any capture) before the first frame."""
        if self.stereo:
            self.ao.OnPreRender()       # one draw of both eyes: single-pass stereo (AO.cs:352-355)
        self.ao.LateUpdate()

    def frame(self, depths: Sequence[torch.Tensor], cameras: Optional[torch.Tensor], render_params: Optional[torch.Tensor] = None):
        """Issues the frame on torch's current stream and returns the new AO: a tensor, or a list for a batch."""
        capturing = torch.cuda.is_current_stream_capturing()
        if self.generation is None and capturing:
            raise RuntimeError(_WARM_UP)
        if cameras is not None:
            self.cameras.copy_(cameras)
        if render_params is not None:
            self.params.copy_(render_params)
        if self.stereo:
            self.ao.OnPreRender()
        linear = self.kind == "linear_f32"
        if self.form == "batch":
            out = self.ao.render_batch(depths, linear=linear)
        else:
            depth = depths[0]
            out = torch.empty(depth.shape, dtype=torch.uint8, device=depth.device)
            if depth.dim() == 3 and depth.shape[0] == 1:
                self.ao.render(depth[0], out[0], linear=linear)
            else:
                self.ao.render(depth, out, linear=linear)
        gen = self.ao._lib.meao_frame_generation(self.ao._ctx)
        if self.generation is None:
            self.generation = gen
        elif gen != self.generation:
            raise RuntimeError(f"meao: a cached context changed under its recorded frames (meao_frame_generation {self.generation} -> "
                               f"{gen}); graphs that hold its frames are stale")
        return out


_CONTEXTS: dict = {}
_WARM_UP = ("meao: the first frame for these inputs must run outside a stream capture -- call the operator once eagerly (a warm-up, as "
            "torch.cuda.graph's recipe and the graph trees of torch.compile do) before capturing it")


def _context(key: tuple) -> _Context:
    ctx = _CONTEXTS.get(key)
    if ctx is None:
        if key[1] >= 0 and torch.cuda.is_current_stream_capturing():
            raise RuntimeError(_WARM_UP)
        ctx = _CONTEXTS[key] = _Context(key)
    return ctx


def contexts() -> dict:
    """The cached contexts, key -> AmbientOcclusion (context_key), for introspection: reservation(), deviceCameraStatus(), deviceParamStatus(),
    kernels_per_frame.  Changing one of them makes its recorded frames stale and the next call raise."""
    return {k: c.ao for k, c in _CONTEXTS.items()}


def release_contexts() -> None:
    """Destroys every cached context and its camera and parameter buffers (after a device synchronise).  The caller's error: calling this while a
    stream capture is open, or while a CUDA graph that holds a frame of one of them is still alive (a torch.cuda.CUDAGraph, or a
    function compiled with mode="reduce-overhead" that has run the operator) -- those graphs would read and write freed memory."""
    if any(c.cameras is not None or c.params is not None for c in _CONTEXTS.values()):
        torch.cuda.synchronize()
    for c in _CONTEXTS.values():
        c.ao.close()
    _CONTEXTS.clear()


# ---- the operators ----------------------------------------------------------------------------------------------------------------
def _key_of(form, depth, layers, kind, cameras, camera, params, reversed_z, projection, layer_projections, variants, hierarchy_depth,
            render_params):
    return context_key(form, depth.device.index if depth.device.index is not None else torch.cuda.current_device(), layers,
                       depth.shape[-2], depth.shape[-1], kind, cameras is not None, camera, params, reversed_z, projection,
                       layer_projections, variants, hierarchy_depth, render_params is not None)


def _check_render_params(render_params: Optional[torch.Tensor], device: torch.device) -> None:
    """render_params: None, or a float32 tensor [2] of (thickness_modifier, intensity) on the depth's device."""
    if render_params is not None and (render_params.device != device or render_params.dtype != torch.float32
                                      or tuple(render_params.shape) != (2,)):
        raise ValueError(f"render_params must be a float32 tensor [2] of (thickness_modifier, intensity) on {device} (got "
                         f"{str(render_params.dtype).replace('torch.', '')} {tuple(render_params.shape)} on {render_params.device})")


@torch.library.custom_op("meao::ambient_occlusion", mutates_args=())
def _ambient_occlusion(depth: torch.Tensor, cameras: Optional[torch.Tensor], camera: Optional[List[float]], kind: str,
                       noise_filter_tolerance: float = 0.0, blur_tolerance: float = -4.6, upsample_tolerance: float = -12.0,
                       thickness_modifier: float = 1.0, intensity: float = 1.0, reversed_z: bool = True, projection: int = 0,
                       layer_projections: Optional[List[int]] = None, single_pass_stereo: bool = False, sample_exhaustively: bool = False,
                       high_quality_mask: int = 0, single_scale: bool = False, hierarchy_depth: int = 4,
                       render_params: Optional[torch.Tensor] = None) -> torch.Tensor:
    L = _frame_layers(depth)
    _check_inputs([depth], L, cameras, camera, kind, projection, layer_projections, single_pass_stereo, high_quality_mask, hierarchy_depth,
                  batch=False)
    _check_render_params(render_params, depth.device)
    key = _key_of("frame", depth, L, kind, cameras, camera,
                  (noise_filter_tolerance, blur_tolerance, upsample_tolerance, thickness_modifier, intensity), reversed_z, projection,
                  layer_projections, (single_pass_stereo, sample_exhaustively, high_quality_mask, single_scale), hierarchy_depth,
                  render_params)
    return _context(key).frame([depth], cameras, render_params)


def _frame_layers(depth: torch.Tensor) -> int:
    if depth.dim() not in (2, 3):
        raise ValueError(f"depth must be [H, W] or [L, H, W] (got {depth.dim()} dimensions)")
    return depth.shape[0] if depth.dim() == 3 else 1


@_ambient_occlusion.register_fake
def _(depth, cameras, camera, kind, noise_filter_tolerance=0.0, blur_tolerance=-4.6, upsample_tolerance=-12.0, thickness_modifier=1.0,
      intensity=1.0, reversed_z=True, projection=0, layer_projections=None, single_pass_stereo=False, sample_exhaustively=False,
      high_quality_mask=0, single_scale=False, hierarchy_depth=4, render_params=None):
    L = _frame_layers(depth)
    _check_inputs([depth], L, cameras, camera, kind, projection, layer_projections, single_pass_stereo, high_quality_mask, hierarchy_depth,
                  batch=False)
    _check_render_params(render_params, depth.device)
    return torch.empty(depth.shape, dtype=torch.uint8, device=depth.device)


@torch.library.custom_op("meao::ambient_occlusion_batch", mutates_args=())
def _ambient_occlusion_batch(depths: List[torch.Tensor], cameras: Optional[torch.Tensor], camera: Optional[List[float]], kind: str,
                             noise_filter_tolerance: float = 0.0, blur_tolerance: float = -4.6, upsample_tolerance: float = -12.0,
                             thickness_modifier: float = 1.0, intensity: float = 1.0, reversed_z: bool = True, projection: int = 0,
                             layer_projections: Optional[List[int]] = None, single_pass_stereo: bool = False,
                             sample_exhaustively: bool = False, high_quality_mask: int = 0, single_scale: bool = False,
                             hierarchy_depth: int = 4, render_params: Optional[torch.Tensor] = None) -> List[torch.Tensor]:
    _check_batch(depths)
    _check_inputs(depths, len(depths), cameras, camera, kind, projection, layer_projections, single_pass_stereo, high_quality_mask,
                  hierarchy_depth, batch=True)
    _check_render_params(render_params, depths[0].device)
    key = _key_of("batch", depths[0], len(depths), kind, cameras, camera,
                  (noise_filter_tolerance, blur_tolerance, upsample_tolerance, thickness_modifier, intensity), reversed_z, projection,
                  layer_projections, (single_pass_stereo, sample_exhaustively, high_quality_mask, single_scale), hierarchy_depth,
                  render_params)
    return _context(key).frame(depths, cameras, render_params)


def _check_batch(depths) -> None:
    if not 1 <= len(depths) <= MAX_BATCH:
        raise ValueError(f"depths must hold 1..{MAX_BATCH} tensors (got {len(depths)})")
    for i, d in enumerate(depths):
        if d.dim() != 2:
            raise ValueError(f"depths[{i}] must be [H, W] (got {d.dim()} dimensions)")


@_ambient_occlusion_batch.register_fake
def _(depths, cameras, camera, kind, noise_filter_tolerance=0.0, blur_tolerance=-4.6, upsample_tolerance=-12.0, thickness_modifier=1.0,
      intensity=1.0, reversed_z=True, projection=0, layer_projections=None, single_pass_stereo=False, sample_exhaustively=False,
      high_quality_mask=0, single_scale=False, hierarchy_depth=4, render_params=None):
    _check_batch(depths)
    _check_inputs(depths, len(depths), cameras, camera, kind, projection, layer_projections, single_pass_stereo, high_quality_mask,
                  hierarchy_depth, batch=True)
    _check_render_params(render_params, depths[0].device)
    return [torch.empty(d.shape, dtype=torch.uint8, device=d.device) for d in depths]


# ---- the Python functions ---------------------------------------------------------------------------------------------------------
Projection = Union[str, int]


def _projection_args(projection: Union[Projection, Sequence[Projection]]):
    """(projection, layer_projections) of the schema from one projection or one per layer ("perspective" / "orthographic" or the
    MeaoProjection values)."""
    def one(p):
        if isinstance(p, str):
            if p not in _PROJECTION_NAMES:
                raise ValueError(f"projection must be one of {sorted(_PROJECTION_NAMES)} (got {p!r})")
            return _PROJECTION_NAMES[p]
        return int(p)
    if isinstance(projection, (str, int)):
        return one(projection), None
    return PERSPECTIVE, [one(p) for p in projection]


def _camera_arg(camera):
    return None if camera is None else [float(c) for c in camera]


def ambient_occlusion(depth: torch.Tensor, cameras: Optional[torch.Tensor] = None, camera: Optional[Sequence[float]] = None,
                      kind: str = "raw_f32", *, noise_filter_tolerance: float = 0.0, blur_tolerance: float = -4.6,
                      upsample_tolerance: float = -12.0, thickness_modifier: float = 1.0, intensity: float = 1.0, reversed_z: bool = True,
                      projection: Union[Projection, Sequence[Projection]] = "perspective", single_pass_stereo: bool = False,
                      sample_exhaustively: bool = False, high_quality_mask: int = 0, single_scale: bool = False,
                      hierarchy_depth: int = 4, render_params: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The AO of one frame (meao::ambient_occlusion): depth [H, W] or [L, H, W] on a CUDA device, of `kind` "raw_f32" / "linear_f32"
    (float32), "d16" (uint16 D16_UNORM codes) or "d24s8" (int32 / uint32 D24_UNORM_S8_UINT words), read in place through its strides
    (last stride 1).  Returns a new contiguous uint8 tensor of the same shape.  Give `cameras` (CUDA float32 [L, 3] of near_clip,
    far_clip, tan_half_fov_h; may change every call) or `camera` (one such triple, fixed).  projection: "perspective", "orthographic",
    or a list with one per layer.  The other keywords are the MeaoParams floats, the Z direction, the MeaoVariants fields and the
    hierarchy depth, with the library's defaults.  render_params: a CUDA float32 tensor [2] of (thickness_modifier, intensity) that may
    change every call; the two keywords are then ignored.  See the module docstring for how contexts are cached."""
    proj, table = _projection_args(projection)
    return torch.ops.meao.ambient_occlusion(depth, cameras, _camera_arg(camera), kind, noise_filter_tolerance, blur_tolerance,
                                            upsample_tolerance, thickness_modifier, intensity, reversed_z, proj, table, single_pass_stereo,
                                            sample_exhaustively, high_quality_mask, single_scale, hierarchy_depth, render_params)


def ambient_occlusion_batch(depths: Sequence[torch.Tensor], cameras: Optional[torch.Tensor] = None,
                            camera: Optional[Sequence[float]] = None, kind: str = "raw_f32", *, noise_filter_tolerance: float = 0.0,
                            blur_tolerance: float = -4.6, upsample_tolerance: float = -12.0, thickness_modifier: float = 1.0,
                            intensity: float = 1.0, reversed_z: bool = True,
                            projection: Union[Projection, Sequence[Projection]] = "perspective", single_pass_stereo: bool = False,
                            sample_exhaustively: bool = False, high_quality_mask: int = 0, single_scale: bool = False,
                            hierarchy_depth: int = 4, render_params: Optional[torch.Tensor] = None) -> List[torch.Tensor]:
    """The AO of a list of [H, W] depths, one layer each, in one layered frame (meao::ambient_occlusion_batch, meao_render_batch): each
    with its own row stride, all of one size, dtype and device; 1..MEAO_MAX_BATCH of them.  Returns one new uint8 [H, W] tensor per
    depth.  The other arguments as ambient_occlusion, with L = len(depths); a per-layer projection list may not hold an orthographic
    entry (the library refuses such tables for batches)."""
    proj, table = _projection_args(projection)
    return torch.ops.meao.ambient_occlusion_batch(list(depths), cameras, _camera_arg(camera), kind, noise_filter_tolerance,
                                                  blur_tolerance, upsample_tolerance, thickness_modifier, intensity, reversed_z, proj, table,
                                                  single_pass_stereo, sample_exhaustively, high_quality_mask, single_scale,
                                                  hierarchy_depth, render_params)
