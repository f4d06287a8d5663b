"""CPU tests of the torch.library operators (miniengineao_b200/torch_ops.py): the fake implementations' shapes, dtypes and refusals on fake
CUDA tensors; one traced graph holding the operator node under make_fx and under Dynamo with fullgraph=True; the schema defaults against
meao_default_params; and the context cache on plan-only contexts: a new value of any keyed field gets its own context, configured with
it, and identical calls share one."""
import ctypes as C

import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode
from torch.fx.experimental.proxy_tensor import make_fx

import harness
import miniengineao_b200
from miniengineao_b200 import _native as N
from miniengineao_b200 import torch_ops as T

CAM = [0.3, 100.0, 0.75]


@pytest.fixture
def fake():
    with FakeTensorMode() as mode:
        yield mode


def _cuda(*shape, dtype=torch.float32):
    return torch.empty(shape, dtype=dtype, device="cuda")


# ---- the fake implementations -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,dtype", [("raw_f32", torch.float32), ("linear_f32", torch.float32), ("d16", torch.uint16),
                                        ("d24s8", torch.int32), ("d24s8", torch.uint32)])
def test_fake_shapes_and_dtypes(fake, kind, dtype):
    for shape in ((90, 160), (1, 90, 160), (6, 90, 160)):
        d = _cuda(*shape, dtype=dtype)
        L = shape[0] if len(shape) == 3 else 1
        for cams in ({"cameras": _cuda(L, 3)}, {"camera": CAM}):
            out = T.ambient_occlusion(d, kind=kind, **cams)
            assert out.shape == d.shape and out.dtype == torch.uint8 and out.device == d.device and out.is_contiguous()
    wide = _cuda(3, 100, 200, dtype=dtype)[:, 5:95, 8:168]                 # a row- and layer-strided view
    out = miniengineao_b200.ambient_occlusion_op(wide, camera=CAM, kind=kind)
    assert out.shape == (3, 90, 160) and out.is_contiguous()
    depths = [_cuda(90, 200, dtype=dtype)[:, :160] for _ in range(4)]
    outs = T.ambient_occlusion_batch(depths, _cuda(4, 3), kind=kind)
    assert len(outs) == 4 and all(o.shape == (90, 160) and o.dtype == torch.uint8 and o.is_contiguous() for o in outs)
    assert len(miniengineao_b200.ambient_occlusion_batch_op(depths[:1], camera=CAM, kind=kind)) == 1


def test_fake_refusals(fake):
    d, c = _cuda(6, 90, 160), _cuda(6, 3)
    cases = [
        (lambda: T.ambient_occlusion(_cuda(90, 160, dtype=torch.float16), camera=CAM), "must be float32"),
        (lambda: T.ambient_occlusion(_cuda(90, 160), camera=CAM, kind="d16"), "must be uint16"),
        (lambda: T.ambient_occlusion(_cuda(90, 160, dtype=torch.int16), camera=CAM, kind="d16"), "must be uint16"),
        (lambda: T.ambient_occlusion(_cuda(90, 160), camera=CAM, kind="d24s8"), "int32 or uint32"),
        (lambda: T.ambient_occlusion(_cuda(90, 160), camera=CAM, kind="f32"), "kind must be one of"),
        (lambda: T.ambient_occlusion(torch.empty(90, 160), camera=CAM), "CUDA tensor"),
        (lambda: T.ambient_occlusion(_cuda(160, 90).t(), camera=CAM), "last-dimension stride of 1"),
        (lambda: T.ambient_occlusion(_cuda(90, 320)[:, ::2], camera=CAM), "last-dimension stride of 1"),
        (lambda: T.ambient_occlusion(d.transpose(1, 2), c), "last-dimension stride of 1"),
        (lambda: T.ambient_occlusion(_cuda(2, 6, 90, 160), c), "[H, W] or [L, H, W]"),
        (lambda: T.ambient_occlusion(d, c, camera=CAM), "exactly one of"),
        (lambda: T.ambient_occlusion(d), "exactly one of"),
        (lambda: T.ambient_occlusion(d, c[:5]), "[6, 3]"),
        (lambda: T.ambient_occlusion(d, _cuda(6, 4)), "[6, 3]"),
        (lambda: T.ambient_occlusion(d, _cuda(6, 3, dtype=torch.float64)), "[6, 3]"),
        (lambda: T.ambient_occlusion(d, torch.empty(6, 3)), "[6, 3]"),
        (lambda: T.ambient_occlusion(d, camera=CAM[:2]), "near_clip, far_clip, tan_half_fov_h"),
        (lambda: T.ambient_occlusion(d, camera=[0.3, 0.2, 1.0]), "far_clip > near_clip"),
        (lambda: T.ambient_occlusion(d, c, projection=["perspective"] * 5), "5 entries for 6 layers"),
        (lambda: T.ambient_occlusion(d, c, projection="fisheye"), "projection must be one of"),
        (lambda: T.ambient_occlusion(d, c, high_quality_mask=16), "high_quality_mask"),
        (lambda: T.ambient_occlusion(d, c, hierarchy_depth=5), "hierarchy_depth"),
        (lambda: T.ambient_occlusion(_cuda(90, 161), camera=CAM, single_pass_stereo=True), "even width"),
        (lambda: T.ambient_occlusion_batch([], camera=CAM), "1..256"),
        (lambda: T.ambient_occlusion_batch([_cuda(9, 16)] * 257, camera=CAM), "1..256"),
        (lambda: T.ambient_occlusion_batch([_cuda(90, 160), _cuda(90, 161)], camera=CAM), "one size"),
        (lambda: T.ambient_occlusion_batch([_cuda(90, 160), _cuda(90, 160, dtype=torch.uint16)], camera=CAM), "must be float32"),
        (lambda: T.ambient_occlusion_batch([_cuda(90, 160), torch.empty(90, 160)], camera=CAM), "CUDA tensor"),
        (lambda: T.ambient_occlusion_batch([_cuda(1, 90, 160)], camera=CAM), "must be [H, W]"),
        (lambda: T.ambient_occlusion_batch([_cuda(90, 160)] * 2, _cuda(3, 3)), "[2, 3]"),
        (lambda: T.ambient_occlusion_batch([_cuda(90, 160)] * 2, camera=CAM, projection=["perspective", "orthographic"]), "batch"),
    ]
    for call, what in cases:
        with pytest.raises(ValueError, match=None) as e:
            call()
        assert what in str(e.value), (what, str(e.value))


# ---- one traced graph -----------------------------------------------------------------------------------------------------------------
def _between_torch_ops(x, cams):
    ao = T.ambient_occlusion(x * 2.0, cams)
    return ao.float() + 1.0


def _batch_between_torch_ops(x, y):
    a, b = T.ambient_occlusion_batch([x + 1.0, y], camera=CAM, intensity=1.1)
    return a.int() - b.int()


def _targets(gm):
    return [n.target for n in gm.graph.nodes if n.op == "call_function"]


def test_make_fx_holds_the_operator():
    with FakeTensorMode():
        x, cams, y = _cuda(90, 160), _cuda(1, 3), _cuda(90, 160)
    gm = make_fx(_between_torch_ops, tracing_mode="fake")(x, cams)
    t = _targets(gm)
    assert torch.ops.meao.ambient_occlusion.default in t
    assert t.index(torch.ops.aten.mul.Tensor) < t.index(torch.ops.meao.ambient_occlusion.default) < t.index(torch.ops.aten.add.Tensor)
    gm = make_fx(_batch_between_torch_ops, tracing_mode="fake")(x, y)
    assert torch.ops.meao.ambient_occlusion_batch.default in _targets(gm)


@pytest.mark.parametrize("fn,op", [(_between_torch_ops, torch.ops.meao.ambient_occlusion),
                                   (_batch_between_torch_ops, torch.ops.meao.ambient_occlusion_batch)])
def test_dynamo_fullgraph_holds_the_operator(fn, op):
    graphs = []

    def record(gm, example_inputs):
        graphs.append(gm)
        return gm.forward

    torch._dynamo.reset()
    with FakeTensorMode():
        a, b = _cuda(90, 160), (_cuda(1, 3) if fn is _between_torch_ops else _cuda(90, 160))
        torch.compile(fn, backend=record, fullgraph=True)(a, b)
    assert len(graphs) == 1
    assert op in _targets(graphs[0])
    torch._dynamo.reset()


def test_schema_defaults_are_the_librarys():
    p = N.MeaoParams()
    N.lib().meao_default_params(C.byref(p))
    schema = torch.ops.meao.ambient_occlusion.default._schema
    default = {a.name: a.default_value for a in schema.arguments}
    for f in ("noise_filter_tolerance", "blur_tolerance", "upsample_tolerance", "thickness_modifier", "intensity"):
        assert T._f32(default[f]) == T._f32(getattr(p, f)), f
    assert default["hierarchy_depth"] == 4 and default["high_quality_mask"] == 0 and default["reversed_z"] is True
    batch = {a.name: a.default_value for a in torch.ops.meao.ambient_occlusion_batch.default._schema.arguments}
    assert {k: v for k, v in batch.items() if k != "depths"} == {k: v for k, v in default.items() if k != "depth"}


# ---- the context cache ----------------------------------------------------------------------------------------------------------------
BASE = dict(form="frame", device=-1, layers=2, height=90, width=160, kind="raw_f32", cameras_on_device=False, camera=CAM,
            params=(0.0, -4.6, -12.0, 1.0, 1.0), reversed_z=True, projection=T.PERSPECTIVE, layer_projections=None,
            variants=(0, 0, 0, 0), hierarchy_depth=4)
CHANGES = {
    "form": "batch", "layers": 3, "height": 92, "width": 162, "kind": "d16", "cameras_on_device": True, "camera": [0.3, 100.0, 0.76],
    "params": (0.0, -4.6, -12.0, 1.0, 1.1), "params_nft": (-1.0, -4.6, -12.0, 1.0, 1.0), "params_bt": (0.0, -4.0, -12.0, 1.0, 1.0),
    "params_ut": (0.0, -4.6, -8.0, 1.0, 1.0), "params_tm": (0.0, -4.6, -12.0, 2.0, 1.0), "reversed_z": False,
    "projection": T.ORTHOGRAPHIC, "layer_projections": [T.PERSPECTIVE, T.ORTHOGRAPHIC], "variants": (1, 0, 0, 0),
    "variants_exh": (0, 1, 0, 0), "variants_hq": (0, 0, 8, 0), "variants_ss": (0, 0, 0, 1), "hierarchy_depth": 2,
}


def _key(**kw):
    return T.context_key(**dict(BASE, **kw))


def _lib_state(ao):
    lib, h = N.lib(), ao._ctx
    p, v, r = N.MeaoParams(), N.MeaoVariants(), N.MeaoReservation()
    lib.meao_get_params(h, C.byref(p))
    lib.meao_get_variants(h, C.byref(v))
    lib.meao_reservation(h, C.byref(r))
    projs = (C.c_int32 * 8)()
    n = lib.meao_get_layer_projections(h, projs, 8)
    cams = (N.MeaoCamera * 8)()
    nc = lib.meao_get_layer_cameras(h, cams, 8)
    return dict(params=tuple(T._f32(getattr(p, f)) for f in ("noise_filter_tolerance", "blur_tolerance", "upsample_tolerance",
                                                              "thickness_modifier", "intensity")),
                variants=(v.single_pass_stereo, v.sample_exhaustively, v.high_quality_mask, v.single_scale),
                depth=lib.meao_get_hierarchy_depth(h), projection=lib.meao_get_projection(h), layer_projections=list(projs[:n]),
                layer_cameras=[(c.near_clip, c.far_clip, c.tan_half_fov_h, c.reversed_z) for c in cams[:nc]],
                zbuffer=tuple(ao.zbuffer_params()), layers=ao.layers, size=(ao._width, ao._height))


def test_context_key_fields():
    T.release_contexts()
    base = T._context(_key())
    assert T._context(_key()) is base
    assert T._context(_key(params=(0.0, float(T._f32(-4.6)), -12.0, 1.0, 1.0))) is base       # the value the library stores
    assert T._context(_key(camera=tuple(CAM))) is base
    seen = {id(base)}
    for name, value in CHANGES.items():
        field = name.split("_")[0] if name.startswith(("params_", "variants_")) else name
        kw = {field: value}
        if field == "cameras_on_device":
            kw["camera"] = None
        ctx = T._context(_key(**kw))
        assert id(ctx) not in seen, name
        seen.add(id(ctx))
        assert T._context(_key(**kw)) is ctx, name
    assert len(T.contexts()) == len(seen)
    T.release_contexts()
    assert T.contexts() == {}


def test_contexts_are_configured_from_their_key():
    T.release_contexts()
    s = _lib_state(T._context(_key()).ao)
    assert s["params"] == tuple(T._f32(x) for x in BASE["params"]) and s["variants"] == (0, 0, 0, 0) and s["depth"] == 4
    assert s["projection"] == T.PERSPECTIVE and s["layer_projections"] == [] and s["layers"] == 2 and s["size"] == (160, 90)
    for kw, check in [
        (dict(params=(-1.0, -4.0, -8.0, 2.0, 1.5)), lambda s: s["params"] == (-1.0, -4.0, -8.0, 2.0, 1.5)),
        (dict(variants=(0, 1, 5, 0)), lambda s: s["variants"] == (0, 1, 5, 0)),
        (dict(variants=(1, 0, 0, 0)), lambda s: s["variants"][0] == 1 and s["size"] == (160, 90)),
        (dict(hierarchy_depth=1), lambda s: s["depth"] == 1),
        (dict(projection=T.ORTHOGRAPHIC), lambda s: s["projection"] == T.ORTHOGRAPHIC),
        (dict(layer_projections=[T.ORTHOGRAPHIC, T.PERSPECTIVE]), lambda s: s["layer_projections"] == [1, 0]
         and len({c for c in s["layer_cameras"]}) == 1),
        (dict(layers=6, form="batch"), lambda s: s["layers"] == 6),
    ]:
        s = _lib_state(T._context(_key(**kw)).ao)
        assert check(s), (kw, s)
    # the host camera: its planes and tan_half_fov_h exactly, and the Z direction -- the constants of a plan given that MeaoCamera
    lib = N.lib()
    for cam, rz in (([0.5, 80.0, 0.625], True), ([0.05, 2000.0, 1.7320508], False), ([0.1, 50.0, 0.3], True)):
        ao = T._context(_key(camera=cam, reversed_z=rz)).ao
        h = C.c_void_p()
        assert lib.meao_create(C.byref(N.MeaoDeviceCfg(-1, 0)), C.byref(h)) == 0
        assert lib.meao_set_camera(h, C.byref(N.MeaoCamera(*cam, int(rz)))) == 0
        assert lib.meao_set_layers(h, 2) == 1 and lib.meao_resize(h, 160, 90) == 1
        assert harness.plan_constants(ao._ctx, 2) == harness.plan_constants(h, 2), cam
        lib.meao_destroy(h)
    # device cameras on a plan-only context: nothing to bind, the host camera stays valid
    assert _lib_state(T._context(_key(cameras_on_device=True, camera=None)).ao)["layers"] == 2
    T.release_contexts()
