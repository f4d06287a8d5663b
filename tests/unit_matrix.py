"""The case matrix of the satellite kernel units -- orthographic (build.py ORTHO_SOURCES), per-layer projections ("mixed",
MIXED_SOURCES), batches (BATCH_SOURCES), layer viewports ("views", VIEW_SOURCES) and device camera tables (CAMERA_SOURCES): one list of
frames that launches every kernel of the five units, with the exact set of those kernels each case must launch.
tests/test_unit_matrix_emulated.py runs it in the CPU emulator, where the launch ledger names the kernels that really ran, counts their
TMA box loads and the CTAs of their grids; tests/test_unit_matrix_gpu.py runs the same cases through libmeao on the GPU.

expected_kernels() is written out from a case's fields, as tests/kernel_matrix.py's is: it does not call the slot functions of
csrc/kernels.h, because it is the independent statement they are checked against.  It names only the five units' kernels; the
perspective prepare of linear ingest, the blend-level upsamples and the render of batch and viewport frames are the core matrix's.

Three kinds of case:
- the slot cases: every depth kind, Z direction, frame form, variant and forced render tile height of each unit, at small sizes;
- the TMA-fed cases, 640 x 360 per layer: every render kernel family (interleaved and wide, checkerboard and exhaustive, tiles
  32 / 16 / 8) of the orthographic, layered orthographic and mixed units, with interior render tiles at every tile height, next to a
  layer boundary in the layered ones;
- the tile-loop cases (persist): every final upsample kernel of the units, plain and premin, in every depth format, at 320 x 180 per
  layer (interior final-level tiles, so the upsample takes TMA), run for three consecutive frames with MEAO_UPS_PERSIST_MIN_WAVES
  tiny, so a CTA walks tiles of different layers and the last CTA's counter re-arm is used by the next frame.  Their layers differ:
  per-layer cameras, mixed projections, targets of their own pitch or misaligned base, viewports at other origins and slices.

And their hostile twins (hostile): the same frames on the depth of tests/hostile_cases.py, each layer salted for its own layer's
camera, so the fast-path guards of every kernel meet zeros, subnormals, infinities, NaNs and the raw depths where the linearisation's
denominator crosses zero: a twin of every slot case, of the TMA-fed render cases and of a few tile-loop cases (whose second frame also
carries a solid hostile block of whole final-level tiles in one layer), the extreme cameras (camera: on layer 0 of a one-layer case,
on the middle layer of a layered one) and the tolerances either side of upsample_fast_div_ok and far below it (params).  A hostile
case compares its float buffers with harness.n_diff(nan_equal=True), the rule of tests/hostile_cases.py; AO codes stay exact.

Every case forces the render tile height (kernels.h kRenderTileHs, MEAO_REN_TILE), so the render kernel a case launches does not
depend on the SM count of the device."""
from __future__ import annotations

from dataclasses import dataclass, replace

import numpy as np

from miniengineao_b200 import Camera
from miniengineao_b200 import _native as N

import harness  # noqa: E402  (tests/ is on sys.path via conftest)
import hostile_cases as HC  # noqa: E402

P, O = N.MEAO_PROJECTION_PERSPECTIVE, N.MEAO_PROJECTION_ORTHOGRAPHIC
TILE_H = (32, 16, 8)                # forced render tile variant 0 / 1 / 2
TMA_FED = (640, 360)                # level 1 is 320 x 180: interior render tiles at every tile height
LOOP_FED = (320, 180)               # interior final-level upsample tiles (the TMA boxes of the tile loop)
FRAMES_PER_LOOP_CASE = 3
KINDS = ("f32", "d16", "d24s8", "linear")
IN = {"f32": 0, "linear": 0, "d16": 1, "d24s8": 2}                 # the raw formats of the kernels' template argument
KIND_CODE = {"f32": 0, "linear": 1, "d16": 2, "d24s8": 3}           # MEAO_DEPTH_*
ARRAY_KINDS = {"f32": "raw_f32", "linear": "linear_f32", "d16": "d16"}
UNITS = ("ortho", "mixed", "batch", "views", "camera")

# (near, far, size) per layer: size is the orthographic half-height (orthographicSize) or the perspective vertical field of view
ORTHO_CAMS = ((0.5, 80.0, 6.0), (1.0, 300.0, 25.0), (0.1, 20.0, 2.0))
MIXED_CAMS = ((0.5, 80.0, 6.0), (1.0, 300.0, 55.0), (0.1, 20.0, 2.0), (0.3, 150.0, 9.0))
PERSP_CAMS = ((0.3, 100.0, 60.0), (0.1, 1000.0, 90.0), (0.5, 50.0, 40.0))
HOSTILE_FED = (203, 97)             # ragged: W % 8 == 3, no level a multiple of 4, 16 or 64
# name -> (near, far, tan_half_fov_h): hostile_cases.CAMERAS with 5 for the default camera's tangent (an orthographic layer's half-width),
# and a half-width small enough that it_i of the orthographic coarse levels overflows to inf
HOSTILE_CAMERAS = {name: (n, f, 5.0 if t is None else t) for name, (n, f, t) in HC.CAMERAS.items()}
HOSTILE_CAMERAS["it_overflows"] = (1.0, 1e30, 1e-10)
# the MeaoParams overrides of hostile_cases.PARAMS either side of upsample_fast_div_ok -> the side their plan must land on
FAST_DIV_SIDE = {("upsample_tolerance", -16.55): True, ("upsample_tolerance", -16.56): False, ("upsample_tolerance", 0.0): True,
                 ("upsample_tolerance", 20.0): False, ("noise_filter_tolerance", 15.65): True, ("noise_filter_tolerance", 15.66): False,
                 ("upsample_tolerance", -37.0): False}
SOLID_BLOCK = (slice(32, 96), slice(64, 192))       # 2 x 2 final-level tiles (64 x 32 outputs) of a tile-loop case's layer 0, frame 1


@dataclass(frozen=True)
class Case:
    unit: str                       # UNITS
    form: str                       # ortho / mixed / camera: "stage" (the final level unfused), "fused" (meao_render), "arrays";
                                    # batch: "arrays", "pointers"; views: "arrays", "pitched"
    layers: int = 1
    table: tuple = ()               # each layer's projection (P / O)
    kind: str = "f32"               # KINDS
    reversed_z: bool = True
    exhaustive: bool = False
    hq: int = 0                     # high_quality_mask
    tile: int = 2                   # forced render tile variant (TILE_H)
    size: tuple = (150, 70)
    persist: bool = False           # the persistent upsample tile loop on every level, FRAMES_PER_LOOP_CASE frames
    hostile: bool = False           # the depth of tests/hostile_cases.py
    camera: str = ""                # a HOSTILE_CAMERAS entry on layer 0 (one layer) or the middle layer (layered); the others keep theirs
    params: tuple = ()              # sorted (name, value) MeaoParams overrides (harness.PARAMS names)

    @property
    def id(self) -> str:
        proj = "".join("O" if p == O else "P" for p in self.table)
        parts = [self.unit, self.form, f"L{self.layers}{proj}", self.kind, "rz" if self.reversed_z else "sz"]
        if self.exhaustive:
            parts.append("exh")
        if self.hq:
            parts.append(f"hq{self.hq}")
        parts += [f"tile{TILE_H[self.tile]}", "x".join(map(str, self.size))]
        if self.persist:
            parts.append("loop")
        if self.hostile:
            parts.append("hostile")
        if self.camera:
            parts.append(self.camera)
        parts += [f"{k}={v}" for k, v in self.params]
        return "-".join(parts)

    @property
    def linear(self) -> bool:
        return self.kind == "linear"

    @property
    def frames(self) -> int:
        return FRAMES_PER_LOOP_CASE if self.persist else 1

    @property
    def tma_fed(self) -> bool:
        return self.size in (TMA_FED, LOOP_FED)

    def buffer_ids(self) -> list:
        """The intermediates to compare with the oracle (ids 1-21); id 17 only where it is the context's own AO."""
        own_ao = self.unit in ("ortho", "mixed", "camera") and self.form != "arrays"
        return [b for b in harness.buffer_ids(self.hq) if own_ao or b != 17]

    @property
    def fast_div_side(self):
        """The side of upsample_fast_div_ok the case's tolerances are chosen for (None: no tolerance override)."""
        sides = {FAST_DIV_SIDE[p] for p in self.params if p in FAST_DIV_SIDE}
        assert len(sides) <= 1, self.id
        return sides.pop() if sides else None

    def cameras(self) -> list:
        W, H = self.size
        rz = self.reversed_z
        if self.unit == "ortho":
            out = [Camera(W, H, nearClipPlane=n, farClipPlane=f, usesReversedZBuffer=rz, orthographic=True, orthographicSize=s)
                   for n, f, s in ORTHO_CAMS[:self.layers]]
        elif self.unit in ("mixed", "camera"):
            out = []
            for l, p in enumerate(self.table):
                n, f, s = MIXED_CAMS[l]
                out.append(Camera(W, H, nearClipPlane=n, farClipPlane=f, usesReversedZBuffer=rz, orthographic=True, orthographicSize=s)
                           if p == O else Camera(W, H, nearClipPlane=n, farClipPlane=f, usesReversedZBuffer=rz, fieldOfView=s))
        else:
            out = [Camera(W, H, nearClipPlane=n, farClipPlane=f, fieldOfView=v, usesReversedZBuffer=rz)
                   for n, f, v in PERSP_CAMS[:self.layers]]
        if self.camera:
            m = 0 if self.layers == 1 else self.layers // 2
            out[m] = hostile_camera(self.camera, W, H, rz, out[m].orthographic)
        return out


def hostile_camera(name: str, W: int, H: int, rz: bool, orthographic: bool) -> Camera:
    """HOSTILE_CAMERAS[name] as an orthographic camera (its planes, its tangent as the half-width) or a perspective one
    (hostile_cases.camera(), or the field of view of the tangent for the cameras hostile_cases has no entry for)."""
    near, far, t = HOSTILE_CAMERAS[name]
    if orthographic:
        return Camera(W, H, nearClipPlane=near, farClipPlane=far, usesReversedZBuffer=rz, orthographic=True, orthographicSize=t / (W / H))
    if name in HC.CAMERAS:
        return HC.camera(name, W, H, rz)
    return Camera(W, H, nearClipPlane=near, farClipPlane=far, usesReversedZBuffer=rz, fieldOfView=HC.fov_for_tan_half_h(t, W, H))


def _ortho(form, L, kind, rz, exh=False, hq=0, tile=2, size=None, persist=False, **hostile):
    return Case("ortho", form, L, (O,) * L, kind, rz, exh, hq, tile, size or ((300, 136) if L == 1 else (150, 70)), persist, **hostile)


def _mixed(form, table, kind, rz, exh=False, hq=0, tile=2, size=None, persist=False, **hostile):
    return Case("mixed", form, len(table), tuple(table), kind, rz, exh, hq, tile, size or ((150, 70) if len(table) == 2 else (120, 56)),
                persist, **hostile)


def _cases() -> list:
    out = []
    kinds = [(k, rz) for k in KINDS for rz in (True, False)]
    arr_kinds = [(k, rz) for k in ("f32", "d16", "linear") for rz in (True, False)]
    # ---- slot cases: every depth kind and Z direction through the stage, fused and fused-premin frames and CUDA arrays
    for L in (1, 3):
        for form, exh, hq in (("fused", False, 0), ("stage", True, 15), ("fused", False, 1)):
            out += [_ortho(form, L, k, rz, exh, hq, i % 3) for i, (k, rz) in enumerate(kinds)]
        out += [_ortho("arrays", L, k, rz, i % 2 == 1, 2 if i < 3 else 0, i % 3) for i, (k, rz) in enumerate(arr_kinds)]
    for table in ((P, O), (O, P, O, O)):
        for form, exh, hq in (("fused", False, 0), ("stage", True, 15), ("fused", False, 1)):
            out += [_mixed(form, table, k, rz, exh, hq, i % 3) for i, (k, rz) in enumerate(kinds)]
        out += [_mixed("arrays", table, k, rz, i % 2 == 1, 2 if i < 3 else 0, i % 3) for i, (k, rz) in enumerate(arr_kinds)]
    # batch and views: the five prepare forms of an array, the seven of a pointer (D24S8 too), both Z directions, the plain and the
    # premin final level of every depth format
    slots = [("arrays", "linear", True, 0), ("arrays", "f32", True, 1), ("arrays", "f32", False, 0), ("arrays", "d16", True, 0),
             ("arrays", "d16", False, 1), ("ptr", "linear", True, 0), ("ptr", "f32", True, 1), ("ptr", "f32", False, 0),
             ("ptr", "d16", True, 0), ("ptr", "d16", False, 1), ("ptr", "d24s8", True, 1), ("ptr", "d24s8", False, 0)]
    for unit, ptr, size, L in (("batch", "pointers", (61, 37), 3), ("views", "pitched", (40, 24), 2)):
        out += [Case(unit, ptr if io == "ptr" else io, L, (P,) * L, k, rz, hq=hq, size=size) for io, k, rz, hq in slots]
    # ---- TMA-fed render cases: each render kernel family of the three render units at every tile height
    for exh in (False, True):
        for t in range(3):
            out.append(_ortho("stage", 1, "f32", True, exh, 15, t, TMA_FED))
            out.append(_ortho("stage", 2, "f32", True, exh, 15, t, TMA_FED))
            out.append(_mixed("stage", (P, O), "f32", True, exh, 15, t, TMA_FED))
    # ---- tile-loop cases: every final upsample kernel of the units, plain and premin, every depth format it has
    for i, (kind, hq) in enumerate((k, hq) for k in ("f32", "d16", "d24s8") for hq in (0, 1)):
        rz = i % 2 == 0
        out.append(_ortho("fused", 1, kind, rz, hq=hq, tile=i % 3, size=LOOP_FED, persist=True))
        out.append(_ortho("fused", 2, kind, rz, hq=hq, tile=i % 3, size=LOOP_FED, persist=True))
        out.append(_mixed("fused", (P, O, P), kind, rz, hq=hq, tile=i % 3, size=LOOP_FED, persist=True))
        out.append(Case("batch", "pointers", 3, (P,) * 3, kind, rz, hq=hq, size=LOOP_FED, persist=True))
        out.append(Case("views", "pitched", 2, (P,) * 2, kind, rz, hq=hq, size=LOOP_FED, persist=True))
    for unit, L in (("batch", 3), ("views", 2)):
        out += [Case(unit, "arrays", L, (P,) * L, k, rz, hq=hq, size=LOOP_FED, persist=True) for k, rz, hq in (("f32", False, 0), ("d16", True, 1))]
    # ---- device camera tables: a bound camera buffer on an orthographic and on a mixed table
    out.append(Case("camera", "fused", 2, (O, O), "f32", True, hq=1, tile=1, size=(97, 61)))
    out.append(Case("camera", "fused", 3, (P, O, P), "d24s8", False, tile=0, size=LOOP_FED))
    return out + _hostile_cases(out)


def _hostile_cases(ordinary: list) -> list:
    out = []
    # ---- hostile twins: every slot case and bound-camera case, every TMA-fed render case, and a tile-loop case of each unit and target
    # form in f32 and in D16
    out += [replace(c, hostile=True) for c in ordinary if not c.persist]
    loops = [c for c in ordinary if c.persist and c.unit != "camera"]
    for unit, form in dict.fromkeys((c.unit, c.form) for c in loops):
        for kind in ("f32", "d16"):
            mine = [c for c in loops if (c.unit, c.form, c.kind) == (unit, form, kind)]
            out.append(replace(mine[0] if kind == "d16" else mine[-1], hostile=True))   # ortho: one layer in D16, two in f32
    # ---- the extreme cameras: raw depth through the stage and the fused frame in both Z directions, D16 / D24S8 under the far / near
    # ratio of 1e7, linear depth under the cameras of extreme tangent; a layered case puts the camera on its middle layer, so the mixed
    # cases take both orders of a [P, O] table for the camera to meet both projections
    HF = HOSTILE_FED
    for i, name in enumerate(HOSTILE_CAMERAS):
        for rz in (True, False):
            for form in ("stage", "fused"):
                out.append(_ortho(form, 1, "f32", rz, hq=9, tile=i % 3, size=HF, hostile=True, camera=name))
                out += [_mixed(form, t, "f32", rz, hq=9, tile=i % 3, size=HF, hostile=True, camera=name) for t in ((P, O), (O, P))]
    for kind in ("d16", "d24s8"):
        for rz in (True, False):
            out.append(_ortho("fused", 1, kind, rz, size=HF, hostile=True, camera="far_near_1e7"))
            out += [_mixed("fused", t, kind, rz, size=HF, hostile=True, camera="far_near_1e7") for t in ((P, O), (O, P))]
    for name in ("tan_half_fov_1em6", "tan_half_fov_1e6", "it_overflows"):
        out.append(_ortho("fused", 1, "linear", True, exh=True, size=HF, hostile=True, camera=name))
        out += [_mixed("fused", t, "linear", True, exh=True, size=HF, hostile=True, camera=name) for t in ((P, O), (O, P))]
    # batches and viewports: every extreme camera on the middle layer, through both target forms
    for i, name in enumerate(HC.CAMERAS):
        kind, rz = ("f32", "d16", "linear", "f32", "d16")[i], i % 2 == 0
        for unit, L, size in (("batch", 3, (61, 37)), ("views", 2, (40, 24))):
            out += [Case(unit, form, L, (P,) * L, kind, rz, size=size, hostile=True, camera=name)
                    for form in (("pointers", "arrays") if unit == "batch" else ("pitched", "arrays"))]
    # ---- the tolerances either side of upsample_fast_div_ok through the fused final level of each unit; one pair of each unit premin
    for u, make in enumerate((lambda kind, rz, hq, j, **kw: _ortho("fused", 1 + j % 2, kind, rz, hq=hq, tile=j % 3, **kw),
                              lambda kind, rz, hq, j, **kw: _mixed("fused", (P, O), kind, rz, hq=hq, tile=j % 3, **kw),
                              lambda kind, rz, hq, j, **kw: Case("batch", "pointers", 3, (P,) * 3, kind, rz, hq=hq, size=(61, 37), **kw),
                              lambda kind, rz, hq, j, **kw: Case("views", "pitched", 2, (P,) * 2, kind, rz, hq=hq, size=(40, 24), **kw))):
        for j, p in enumerate(FAST_DIV_SIDE):
            out.append(make(("f32", "d16", "d24s8")[(j + u) % 3], j % 2 == 0, int(j // 2 == u % 3), j, hostile=True, params=(p,)))
    return out


CASES = _cases()


def _b(v: bool) -> str:
    return "true" if v else "false"


def expected_kernels(c: Case) -> set:
    """The five units' kernels (emu's names, 'render_ao_ortho_kernel<0, true, 32>') case `c` launches, each at least once."""
    raw = not c.linear
    fmt = IN[c.kind]
    pre = "premin_" if c.hq & 1 else ""
    out = set()
    if c.unit in ("batch", "views"):
        u = "batch" if c.unit == "batch" else "views"
        if c.form == "arrays":
            out.add(f"prepare_depth_array_{u}_kernel<{_b(raw)}, {_b(c.reversed_z or not raw)}, {fmt}>")
            out.add(f"blur_upsample_{pre}array_{u}_kernel<false, true>")
        else:
            out.add(f"prepare_depth_low_{u}_kernel<{_b(raw)}, {_b(c.reversed_z or not raw)}, {fmt}>")
            out.add(f"blur_upsample_{pre}lin_{u}_kernel<{fmt}, false, true>")
        return out
    # the render units: a uniform orthographic table takes the orthographic kernels, any other the mixed ones; a bound camera buffer
    # adds the camera stage
    mixed = len(set(c.table)) > 1
    if c.unit == "camera":
        out.add("camera_tables_mixed_kernel" if mixed else "camera_tables_kernel")
    layered = c.layers > 1 or c.unit == "camera"
    u = "mixed_layered" if mixed else ("ortho_layered" if layered else "ortho")
    if raw:                                             # linear ingest keeps the perspective prepare
        if c.form == "arrays":
            out.add(f"prepare_depth_array_{'mixed' if mixed else 'ortho'}_kernel<true, {_b(c.reversed_z)}, {fmt}>")
        else:
            out.add(f"prepare_depth{'_low' if c.form == 'fused' else ''}_{u}_kernel<true, {_b(c.reversed_z)}, {fmt}>")
    th = TILE_H[c.tile]
    out.add(f"render_ao_{u}_kernel<0, {_b(c.exhaustive)}, {th}>")
    if c.hq:
        out.add(f"render_ao_{u}_kernel<1, {_b(c.exhaustive)}, {th}>")
    if raw and c.form == "fused":                       # the fused final level of raw depth
        out.add(f"blur_upsample_{pre}lin_{'mixed' if mixed else u}_kernel<{fmt}, false, true>")
    return out


def upsample_kernel(c: Case) -> str:
    """The unit's final upsample kernel of case `c` (the one a tile-loop case exists for)."""
    ups = [k for k in expected_kernels(c) if k.startswith("blur_upsample")]
    assert len(ups) == 1, (c.id, ups)
    return ups[0]


def depth(c: Case, frame: int = 0):
    """(the depth of every layer in the case's ingest format [layers, H, W], the float32 the oracle sees); each frame of a tile-loop
    case its own."""
    if c.hostile:
        return _hostile_depth(c, frame)
    W, H = c.size
    if c.unit in ("ortho", "mixed", "camera"):
        seed = c.tile + 3 * c.layers + 101 * frame
        if c.linear:
            d = harness.contrasting_layers(W, H, c.layers, seed=seed)
            return d, d
        return harness.ingest(harness.frames(W, H, c.layers, seed=seed, reversed_z=c.reversed_z), c.kind)
    seed = {"arrays": 1, "pointers": 2, "pitched": 7}[c.form] + 101 * frame
    lin = harness.contrasting_layers(W, H, c.layers, seed=seed)
    if c.linear:
        return lin, lin
    return harness.ingest(harness.raw(lin, reversed_z=c.reversed_z), c.kind)


def _hostile_depth(c: Case, frame: int):
    """Hostile depth of every layer, raw f32 salted with the values where its own layer's linearisation crosses zero (the zbuffer params
    of that layer's camera, orthographic or perspective); a seed of its own per layer and frame.  Frame 1 (the second frame of a
    tile-loop case) also fills SOLID_BLOCK of layer 0 with one value -- NaN, +inf, -inf, or the sky code of a UNORM format -- so whole
    tiles of one layer are hostile while the next layer's are not: a CTA that carries a box, a border or a count from one tile to the
    next shows."""
    W, H = c.size
    ds, seen = [], []
    for l, cam in enumerate(c.cameras()):
        seed = 7 * l + 101 * frame + 3 * c.layers + c.tile + 13 * KIND_CODE[c.kind]
        if c.kind == "linear":
            d = s = HC.hostile_linear(W, H, seed=seed)
        elif c.kind == "f32":
            d = s = HC.hostile_raw(W, H, harness.context(cam).zbuffer_params(), c.reversed_z, seed=seed)
        else:
            d, s = HC.hostile_unorm(W, H, 16 if c.kind == "d16" else 24, c.reversed_z, seed=seed)
        ds.append(d)
        seen.append(s)
    d, seen = np.stack(ds), np.stack(seen)
    if frame == 1:
        if c.kind in ("f32", "linear"):
            d[(0,) + SOLID_BLOCK] = seen[(0,) + SOLID_BLOCK] = (np.nan, np.inf, -np.inf)[(c.hq + c.layers + c.reversed_z) % 3]
        else:
            full = (1 << (16 if c.kind == "d16" else 24)) - 1
            code = 0 if c.reversed_z else full                                  # the sky of the Z direction
            blk = d[(0,) + SOLID_BLOCK]
            d[(0,) + SOLID_BLOCK] = (blk & ~np.array(full, blk.dtype)) | np.array(code, blk.dtype)
            seen[(0,) + SOLID_BLOCK] = np.float32(code) * np.float32(1.0 / full)
    return d, seen


def oracle(c: Case, cam, threads=4):
    """The oracle of one layer of case `c` with camera `cam`: the orthographic one for an orthographic camera, else the perspective one."""
    kw = dict(sample_exhaustively=c.exhaustive, high_quality_mask=c.hq, **dict(c.params))
    if cam.orthographic:
        from ortho_oracle import OrthoOracle
        return OrthoOracle(cam.pixelWidth, cam.pixelHeight, near=cam.nearClipPlane, far=cam.farClipPlane,
                           tan_half_fov_h_=1.0 / cam.projection00, reversed_z=cam.usesReversedZBuffer, linear=c.linear, threads=threads, **kw)
    return harness.oracle(cam.pixelWidth, cam.pixelHeight, camera=cam, linear=c.linear, threads=threads, **kw)


# ---- the targets of batch and viewport cases ---------------------------------------------------------------------------------------
def batch_pointer_layout(c: Case) -> list:
    """Per layer (depth row pitch in elements, depth base offset in elements, AO row pitch in bytes, AO base offset in bytes): layer 0
    tight and aligned, layer 1 at an odd row pitch, layer 2 at a base that misses the vector alignment."""
    W = c.size[0]
    return [(W, 0, W, 0), (W + 3, 0, W + 5, 0), (W, 1, W + 1, 3)][:c.layers]


def batch_array_layout(c: Case) -> list:
    """Per layer (depth array extent (h, w), depth shape, AO shape): exact-size 2-D arrays, oversized 2-D ones, an oversized layered one
    of one layer."""
    W, H = c.size
    ext = [(H, W), (H + 3, W + 5), (H + 1, W + 2)]
    shapes = ["2d", "2d", "layered"]
    return [(ext[l], shapes[l], shapes[c.layers - 1 - l]) for l in range(c.layers)]


def view_arrays_layout(c: Case) -> tuple:
    """(table, depth shape, depth extent (slices, h, w), AO shape, AO extent) of an array viewport case: the slot cases side by side
    in one 2-D array; the tile-loop cases at other origins and other slices of layered arrays."""
    W, H = c.size
    if not c.persist:
        return [(0, 0, 0, 0, 0, 0), (W, 0, 0, W, 0, 0)], "2d", (1, H, 2 * W), "2d", (1, H, 2 * W)
    return [(5, 3, 1, 0, 0, 1), (0, 0, 0, 3, 1, 0)], "layered", (2, H + 3, W + 5), "layered", (2, H + 1, W + 3)


def view_pitched_layout(c: Case) -> tuple:
    """(table, depth row, depth slice (elements), AO row, AO slice (bytes), slices) of a pointer viewport case: the slot cases side by
    side in one slice; the tile-loop cases in two slices, layer 1's depth at an odd column (a misaligned base) and row."""
    W, H = c.size
    if not c.persist:
        return [(0, 0, 0, 0, 0, 0), (W, 0, 0, W, 0, 0)], 2 * W, 2 * W * H, 2 * W, 2 * W * H, 1
    drow, arow = 2 * W + 16, 2 * W + 8
    return [(0, 0, 0, W + 3, 0, 1), (W + 1, 1, 1, 0, 2, 0)], drow, drow * (H + 2), arow, arow * (H + 3), 2


def loop_tiles(c: Case) -> int:
    """The tiles of the final upsample of case `c` (64 x 32 outputs each, every layer's): a launch without the tile loop has one CTA
    per tile."""
    W, H = c.size
    return -(-W // 64) * -(-H // 32) * c.layers
