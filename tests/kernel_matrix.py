"""The kernel case matrix: one list of frames (and calls of the other kernel units) that launches every entry of every kernel table,
with the exact set of kernels each case must launch.  tests/test_kernel_matrix_emulated.py runs it in the CPU emulator, where a
launch ledger names the kernels that really ran; tests/test_kernel_matrix_gpu.py runs its frames through libmeao on the GPU.

expected_kernels() is written out from a case's fields -- it does not call the slot functions of csrc/kernels.h (prepare_slot,
render_slot, upsample_slot, depth_format_slot), because it is the independent statement those functions and the MEAO_*_SLOTS tables
are checked against: a table entry swapped with another still compiles, loads and counts the same, but launches the wrong kernel.

Every frame case forces the render tile height (kernels.h kRenderTileHs, Frame(render_tile=) / MEAO_REN_TILE), so the render kernel a
case launches does not depend on the SM count of the device."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from test_layers_emulated import _raw, contrasting_layers  # noqa: E402  (tests/ is on sys.path via conftest)

KINDS = ("linear", "f32", "d16", "d24s8")
TILE_H = (32, 16, 8)                # forced render tile variant 0 / 1 / 2
RAGGED, TMA_FED = (161, 93), (640, 360)     # no level a multiple of 4, 16 or 64; level 1 has interior (TMA-fed) tiles at every tile height


@dataclass(frozen=True)
class Case:
    form: str                       # "stage": prepare -> LinearDepth -> render -> upsample, the final level unfused; "fused": meao_render;
                                    # "arrays": CUDA arrays; the other units: "composite", "debug_view", "debug_composite", "halo", "band_exchange"
    layers: int = 1
    kind: str = "f32"               # KINDS
    reversed_z: bool = True
    exhaustive: bool = False
    hq: int = 0                     # high_quality_mask
    single_scale: bool = False
    tile: int = 2                   # forced render tile variant (TILE_H)
    size: tuple = RAGGED

    @property
    def id(self) -> str:
        if self.form not in ("stage", "fused", "arrays"):
            return self.form
        parts = [self.form, f"L{self.layers}", self.kind]
        if self.kind != "linear":
            parts.append("rz" if self.reversed_z else "sz")
        if self.exhaustive:
            parts.append("exh")
        if self.hq:
            parts.append(f"hq{self.hq}")
        if self.single_scale:
            parts.append("single")
        parts += [f"tile{TILE_H[self.tile]}", "x".join(map(str, self.size))]
        return "-".join(parts)

    @property
    def frame(self) -> bool:
        return self.form in ("stage", "fused", "arrays")

    def oracle_kw(self) -> dict:
        kw = dict(intensity=1.1, reversed_z=self.reversed_z, high_quality_mask=self.hq, sample_exhaustively=self.exhaustive)
        if self.kind == "linear":
            kw["depth_is_linear"] = True
        if self.single_scale:
            kw["single_scale"] = True
        return kw

    def buffer_ids(self) -> list:
        """The intermediates a frame of this case produces (and the AO): debug ids 1-17, 18-21 for its high-quality levels."""
        if self.single_scale:
            return [1, 2, 3, 4, 5, 10, 17]
        return list(range(1, 18)) + [17 + k for k in range(1, 5) if (self.hq >> (k - 1)) & 1]


def _cases() -> list:
    out = []
    # prepare: every depth kind (linear depth has one kernel for both Z directions) through both frame forms, 1 and 3 layers
    kinds = [("linear", True)] + [(k, rz) for k in KINDS[1:] for rz in (True, False)]
    for form in ("stage", "fused"):
        for layers in (1, 3):
            out += [Case(form, layers, k, rz) for k, rz in kinds]
    # the fused final level with high_quality_mask bit 0 (the premin kernels) on every raw depth format
    out += [Case("fused", layers, k, hq=1) for layers in (1, 3) for k in KINDS[1:]]
    # arrays: every kind a CUDA array holds (no D24S8), layered; one 2-D frame with the premin final level
    out += [Case("arrays", 3, k, rz) for k, rz in kinds if k != "d24s8"] + [Case("arrays", 1, "f32", hq=1)]
    # render: the wide kernel at every level (hq 15) and the interleaved one, checkerboard and exhaustive sampling, every tile height
    out += [Case("stage", layers, "f32", exhaustive=exh, hq=15, tile=t, size=TMA_FED) for layers in (1, 3) for exh in (False, True)
            for t in range(3)]
    out.append(Case("stage", 1, "f32", single_scale=True))
    out += [Case(u) for u in ("composite", "debug_view", "debug_composite", "halo", "band_exchange")]
    return out


CASES = _cases()
FRAME_CASES = [c for c in CASES if c.frame]


def _b(v: bool) -> str:
    return "true" if v else "false"


def _prepare(c: Case) -> str:
    raw = c.kind != "linear"
    fmt = {"linear": 0, "f32": 0, "d16": 1, "d24s8": 2}[c.kind]
    base = {"stage": "prepare_depth", "fused": "prepare_depth_low", "arrays": "prepare_depth_array"}[c.form]
    if c.layers > 1 and c.form != "arrays":
        base += "_layered"
    return f"{base}_kernel<{_b(raw)}, {_b(c.reversed_z or not raw)}, {fmt}>"


def expected_kernels(c: Case) -> set:
    """The names (emu.kernel_ledger's form, 'render_ao_kernel<0, true, 32>') of the kernels case `c` launches, each at least once."""
    if not c.frame:
        return {"composite": {"composite_kernel<false>", "composite_kernel<true>"},
                "debug_view": {"debug_view_kernel", "synth_tiled_kernel"},
                "debug_composite": {"debug_composite_kernel<false>", "debug_composite_kernel<true>"},
                "halo": {"halo_copy_kernel"},
                "band_exchange": {"band_exchange_kernel"}}[c.form]
    layered = c.layers > 1
    levels = [1] if c.single_scale else [1, 2, 3, 4]
    out = {_prepare(c)}
    ren = "render_ao_layered_kernel" if layered else "render_ao_kernel"
    out.add(f"{ren}<0, {_b(c.exhaustive)}, {TILE_H[c.tile]}>")
    if any((c.hq >> (k - 1)) & 1 for k in levels):
        out.add(f"{ren}<1, {_b(c.exhaustive)}, {TILE_H[c.tile]}>")
    ups = "_layered" if layered else ""
    for lo in levels[1:]:               # the blend levels 4 -> 3 -> 2 -> 1: a hi-res AO, f32 hi-res depth
        out.add(f"blur_upsample{'_premin' if (c.hq >> (lo - 1)) & 1 else ''}{ups}_kernel<true, false>")
    premin = "_premin" if c.hq & 1 else ""
    if c.form == "stage":               # the final level: no hi-res AO, LinearDepth (f16) as the hi-res depth
        out.add(f"blur_upsample{premin}{ups}_kernel<false, true>")
    elif c.form == "arrays":
        out.add(f"blur_upsample{premin}_array_kernel<false, true>")
    else:
        fmt = {"linear": 0, "f32": 0, "d16": 1, "d24s8": 2}[c.kind]
        out.add(f"blur_upsample{premin}_lin{ups}_kernel<{fmt}, false, true>")
    return out


def depth(c: Case):
    """(depth in the case's ingest format, [layers, H, W]; the float32 the oracle sees per layer).  contrasting_layers with a sky patch
    in layer 2, and in layer 0 of a single-layer frame; native codes carry stencil bits."""
    W, H = c.size
    lin = contrasting_layers(W, H, c.layers, seed=W + c.layers)
    if c.kind == "linear":
        return lin, lin
    raw = _raw(lin, reversed_z=c.reversed_z)
    if c.layers == 1:
        raw[0, H // 4: H // 2, W // 5: W // 2] = 0.0
    if c.kind == "f32":
        return raw, raw
    bits = 16 if c.kind == "d16" else 24
    full = (1 << bits) - 1
    codes = np.clip(np.rint(raw.astype(np.float64) * full), 0, full).astype(np.uint32)
    as_float = (codes.astype(np.float32) * np.float32(1.0 / full)).astype(np.float32)
    words = codes.astype(np.uint16) if bits == 16 else codes | (np.uint32(0xA5) << np.uint32(24))
    return words, as_float
