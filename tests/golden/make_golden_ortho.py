"""Generates tests/golden/ortho/*.npz from the orthographic oracle (tests/ortho_oracle.py), as make_golden.py does for perspective
frames.  Self-generated like those: they pin the orthographic oracle against regressions and let the GPU tests compare against
committed bytes without running the oracle.  A directory of their own, so the perspective fixture tests never read them.  Re-run:
    python tests/golden/make_golden_ortho.py
Keys: depth (raw, reversed Z unless camera[3] == 0), camera = [near, far, orthographicSize, reversed_z], params (MeaoParams floats),
ao, buf<id> for ids 1-17 (unorm8 codes, f16 for LinearDepth and TiledDepth, f32 for LowDepth)."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from miniengineao_b200 import Camera, synth  # noqa: E402
from ortho_oracle import OrthoOracle  # noqa: E402

CASES = {
    # name: (W, H, eye depth / far generator, near, far, orthographicSize, reversed_z, intensity)
    "ortho_corridor_160x90": (160, 90, lambda: synth.corridor(160, 90), 0.5, 80.0, 6.0, True, 1.1),
}


def raw_depth(lin, near, far, reversed_z):
    """Raw orthographic depth whose linearisation is close to `lin` (eye depth / far, clamped into [near / far, 1])."""
    r = np.float64(np.float32(near) / np.float32(far))
    lin = np.clip(lin.astype(np.float64), r, 1.0)
    d = (1.0 - lin) / (1.0 - r) if reversed_z else (lin - r) / (1.0 - r)
    return np.clip(d, 0.0, 1.0).astype(np.float32)


def main():
    os.makedirs(os.path.join(HERE, "ortho"), exist_ok=True)
    for name, (W, H, gen, near, far, size, rz, intensity) in CASES.items():
        cam = Camera(W, H, nearClipPlane=near, farClipPlane=far, usesReversedZBuffer=rz, orthographic=True, orthographicSize=size)
        depth = raw_depth(gen(), near, far, rz)
        o = OrthoOracle(W, H, near=near, far=far, tan_half_fov_h_=1.0 / cam.projection00, reversed_z=rz, intensity=intensity)
        ao = o.run(depth)
        data = {"depth": depth, "ao": ao, "camera": np.array([near, far, size, int(rz)], np.float32),
                "params": np.array([0.0, -4.6, -12.0, 1.0, intensity], np.float32)}
        for bid in range(1, 18):
            b = o.buffer(bid)
            data[f"buf{bid}"] = o.codes(bid) if bid >= 10 else (b.astype(np.float16) if bid == 1 or 6 <= bid <= 9 else b.copy())
        np.savez_compressed(os.path.join(HERE, "ortho", name + ".npz"), **data)
        print(name, W, H, "ao mean", ao.mean())


if __name__ == "__main__":
    main()
