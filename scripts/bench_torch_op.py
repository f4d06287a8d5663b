"""The AO frame under torch.compile, on one GPU, with cameras that move on every call.  Per size (1920x1080, 3840x2160) and layer count
(1, 6), four arms alternated in one process (so all see the same clocks and neighbours), medians over rounds:
  (a) AmbientOcclusion.render, its bound camera tensor written with copy_ before each call;
  (b) the eager operator, miniengineao_b200.torch_ops.ambient_occlusion(depth, cameras);
  (c) a function that calls the operator, compiled with mode="reduce-overhead": the graph trees replay the recorded frame, with the
      call's cameras copied into the graph's input and then into the context's camera buffer;
  (d) the same function with the AO call (a) as a graph break, compiled the same way: what a torch.compile user gets without the operator.
The depth is one static tensor (torch._dynamo.mark_static_address, so the graph trees do not copy it); each call gets a camera tensor
already on the device.  For each arm: device microseconds per frame (CUDA events around the frames) and host microseconds per call (the
issue loop, before the final synchronise).  After the timed rounds every arm renders the same cameras once and the AO is compared.  Prints
the card name and power limit with the numbers; writes nothing in the tree (the compiler's caches go to a temporary directory).

    python scripts/bench_torch_op.py [--rounds 7] [--frames 100]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("TORCHINDUCTOR_CACHE_DIR", tempfile.mkdtemp(prefix="meao_inductor_"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from miniengineao_b200 import AmbientOcclusion, Camera, synth  # noqa: E402
from miniengineao_b200 import torch_ops as T  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def camera_rows(W, H, L, i):
    """The cameras of call i: planes and a field of view that move every call."""
    rows = []
    for l in range(L):
        c = Camera(W, H, nearClipPlane=0.3 + 0.01 * ((i + l) % 7), farClipPlane=1000.0 - (i % 5), fieldOfView=55.0 + 0.5 * ((i + 3 * l) % 11))
        rows.append((c.nearClipPlane, c.farClipPlane, 1.0 / c.projection00))
    return rows


def bench(W, H, L, rounds, frames):
    raw = np.stack([synth.lin01_to_raw(synth.corridor(W, H, frame=i)).astype(np.float32) for i in range(L)])
    depth = torch.from_numpy(raw if L > 1 else raw[0]).cuda()
    torch._dynamo.mark_static_address(depth)
    cams = [torch.tensor(camera_rows(W, H, L, i), dtype=torch.float32, device="cuda") for i in range(frames)]

    ao = AmbientOcclusion(Camera(W, H, nearClipPlane=0.3, farClipPlane=1000.0), device=0)
    ao.layers = L
    ao.deviceCameras = torch.empty((L, 3), dtype=torch.float32, device="cuda")

    def render(d, c):
        ao.deviceCameras.copy_(c)
        return ao.render(d)

    def with_op(d, c):
        return T.ambient_occlusion(d, c)

    render_outside_the_graph = torch._dynamo.disable(render)     # the graph break Dynamo makes at the ctypes call

    def with_graph_break(d, c):
        return render_outside_the_graph(d, c)

    compiled_op = torch.compile(with_op, mode="reduce-overhead", fullgraph=True)
    compiled_break = torch.compile(with_graph_break, mode="reduce-overhead")

    def stepped(fn):
        def call(d, c):
            torch.compiler.cudagraph_mark_step_begin()
            return fn(d, c)
        return call

    arms = {"a_render": render, "b_eager_op": with_op, "c_compiled_op": stepped(compiled_op), "d_compiled_graph_break": stepped(compiled_break)}
    for fn in arms.values():
        for i in range(3):
            fn(depth, cams[i])
    torch.cuda.synchronize()
    dev = {n: [] for n in arms}
    host = {n: [] for n in arms}
    for _ in range(rounds):
        for name, fn in arms.items():
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            t0.record()
            h0 = time.perf_counter()
            for i in range(frames):
                fn(depth, cams[i])
            h1 = time.perf_counter()
            t1.record()
            t1.synchronize()
            dev[name].append(1000.0 * t0.elapsed_time(t1) / frames)
            host[name].append(1e6 * (h1 - h0) / frames)
    outs = {name: fn(depth, cams[frames - 1]).cpu() for name, fn in arms.items()}
    equal = all(torch.equal(outs["a_render"], o) for o in outs.values())
    res = {"size": f"{W}x{H}", "layers": L, "rounds": rounds, "frames_per_round": frames, "ao_equal_between_arms": equal,
           "device_us_per_frame_median": {n: round(statistics.median(v), 1) for n, v in dev.items()},
           "host_us_per_call_median": {n: round(statistics.median(v), 1) for n, v in host.items()},
           "device_us_per_frame_rounds": {n: [round(x, 1) for x in v] for n, v in dev.items()}}
    ao.close()
    torch._dynamo.reset()           # drops the graph trees that hold frames of the operator's context before it is released
    T.release_contexts()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--frames", type=int, default=100)
    ap.add_argument("--sizes", default="1920x1080,3840x2160")
    ap.add_argument("--layers", default="1,6")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_torch_op.py needs a CUDA device")
    res = {"card": card(), "torch": torch.__version__, "results": []}
    for size in a.sizes.split(","):
        W, H = (int(v) for v in size.split("x"))
        for L in (int(x) for x in a.layers.split(",")):
            res["results"].append(bench(W, H, L, a.rounds, a.frames))
            print(json.dumps(res["results"][-1]), flush=True)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
