"""The component entry points of the C-ABI (the calls the parity tests probe the device with) refuse what they cannot run -- an
uncommitted scene, an out-of-range id or `what`, a null array -- with B2_ERR_INVALID and a message, and succeed on zero items."""
import ctypes as C

import numpy as np
import pytest

from mitsuba_b200 import api
from mitsuba_b200.scene import cornell_box, envmap_scene, smoke_scene, textured_scene

pytestmark = pytest.mark.gpu
B2_OK, B2_ERR_INVALID = 0, 1
N = 4  # items of a refused call: every array it is given is large enough


def _p(a):
    return a.ctypes.data_as(C.POINTER(C.c_float)) if a is not None else None


def _rays(n):
    r = np.zeros((n, 8), np.float32)
    r[:, 0:3] = (278.0, 273.0, -800.0)  # from the Cornell camera into the box
    r[:, 3] = 1e-4
    r[:, 6] = 1.0
    r[:, 7] = 1e30
    return r


def _uv(n):
    return np.full((n, 2), 0.25, np.float32)


# entry point -> (scene, {array: (width, required, initial value)}, call(L, handle, n, arrays, **overrides)).  Arrays are built with
# max(n, 1) rows, so a call with n = 0 gets real pointers.
ENTRIES = {
    "b2_trace": ("cornell", {"rays": (8, True, _rays), "t": (1, False, 0), "u": (1, False, 0), "v": (1, False, 0), "prim": (1, False, 0)},
                 lambda L, h, n, a: L.b2_trace(h, C.c_uint64(n), _p(a["rays"]), C.c_int(0), C.c_int(1), _p(a["t"]), _p(a["u"]), _p(a["v"]),
                                               _p(a["prim"]), None)),
    "b2_bsdf_eval": ("cornell", {"wi": (3, True, 0.5), "wo": (3, True, 0.5), "rgb": (3, True, 0), "pdf": (1, True, 0)},
                     lambda L, h, n, a, mat=0: L.b2_bsdf_eval(h, C.c_int(mat), C.c_uint64(n), _p(a["wi"]), _p(a["wo"]), C.c_int(1),
                                                              _p(a["rgb"]), _p(a["pdf"]))),
    "b2_bsdf_sample": ("cornell", {"wi": (3, True, 0.5), "samples": (3, True, 0.5), "out": (10, True, 0)},
                       lambda L, h, n, a, mat=0: L.b2_bsdf_sample(h, C.c_int(mat), C.c_uint64(n), _p(a["wi"]), _p(a["samples"]), C.c_int(1),
                                                                  _p(a["out"]))),
    "b2_sample_emitter_direct": ("cornell", {"ref": (6, True, 0.5), "samples": (2, True, 0.5), "out": (12, True, 0)},
                                 lambda L, h, n, a: L.b2_sample_emitter_direct(h, C.c_uint64(n), _p(a["ref"]), _p(a["samples"]), C.c_int(1),
                                                                               _p(a["out"]))),
    "b2_medium_probe": ("smoke", {"in": (8, True, 0.5), "out": (3, True, 0)},
                        lambda L, h, n, a, medium=0, what=0: L.b2_medium_probe(h, C.c_int(medium), C.c_int(what), C.c_uint64(n), _p(a["in"]),
                                                                               C.c_uint64(1), C.c_int(1), _p(a["out"]))),
    "b2_texture_eval": ("textured", {"uv": (2, True, _uv), "partials": (4, False, 0.01), "out": (3, True, 0)},
                        lambda L, h, n, a, tex=0: L.b2_texture_eval(h, C.c_int(tex), C.c_uint64(n), _p(a["uv"]), _p(a["partials"]), C.c_int(1),
                                                                    _p(a["out"]))),
    "b2_envmap_probe": ("envmap", {"in": (3, True, 0.5), "out": (3, True, 0)},
                        lambda L, h, n, a, what=0: L.b2_envmap_probe(h, C.c_int(what), C.c_uint64(n), _p(a["in"]), C.c_int(1), _p(a["out"]))),
    "b2_texture_partials": ("textured", {"pos_hit": (6, True, 0.5), "out": (6, True, 0)},
                            lambda L, h, n, a: L.b2_texture_partials(h, C.c_uint64(n), _p(a["pos_hit"]), C.c_int(4), C.c_int(1), _p(a["out"]))),
    "b2_camera_rays": ("cornell", {"pos": (2, True, 0.5), "rays": (8, True, 0)},
                       lambda L, h, n, a: L.b2_camera_rays(h, C.c_uint64(n), _p(a["pos"]), C.c_int(1), _p(a["rays"]))),
    # n = the number of dimensions
    "b2_sampler_stream": ("cornell", {"out": (1, True, 0)},
                          lambda L, h, n, a: L.b2_sampler_stream(h, C.c_int(0), C.c_uint64(1), C.c_int(4), C.c_int(1), C.c_int(2), C.c_int(0),
                                                                 C.c_int(n), _p(a["out"]))),
}
# bad ids and `what` values -> the message they are refused with
BAD = {
    "b2_bsdf_eval": [({"mat": 99}, "invalid material id"), ({"mat": -1}, "invalid material id")],
    "b2_bsdf_sample": [({"mat": 99}, "invalid material id")],
    "b2_medium_probe": [({"medium": 5}, "invalid medium id"), ({"what": 4}, "b2_medium_probe: invalid argument")],
    "b2_texture_eval": [({"tex": 7}, "invalid texture id")],
    "b2_envmap_probe": [({"what": 3}, "b2_envmap_probe: invalid argument")],
}
SENTINEL = 7.0


@pytest.fixture(scope="module")
def scenes(b2ctx):
    out = {"cornell": api.Scene(b2ctx, cornell_box(16, 16)),
           "textured": api.Scene(b2ctx, textured_scene(16, 16, tex_res=16, n_theta=8, n_phi=16)),
           "smoke": api.Scene(b2ctx, smoke_scene(16, 16, res=8)),
           "envmap": api.Scene(b2ctx, envmap_scene(16, 16, map_width=32, n_theta=8, n_phi=16))}
    yield out
    for s in out.values():
        s.close()


def arrays(spec, n):
    a = {}
    for name, (w, _, init) in spec.items():
        a[name] = init(max(n, 1)) if callable(init) else np.full((max(n, 1), w), init, np.float32)
    return a


def refused(ctx, rc, message):
    assert rc == B2_ERR_INVALID
    assert message in ctx.err()


@pytest.mark.parametrize("entry", sorted(ENTRIES))
def test_uncommitted_scene_is_refused(b2ctx, entry):
    _, spec, call = ENTRIES[entry]
    h = C.c_void_p()
    assert b2ctx.L.b2_scene_create(b2ctx.h, C.byref(h)) == B2_OK
    try:
        refused(b2ctx, call(b2ctx.L, h, N, arrays(spec, N)), "scene not committed")
    finally:
        b2ctx.L.b2_scene_destroy(h)


@pytest.mark.parametrize("entry", sorted(ENTRIES))
def test_null_required_array_is_refused(b2ctx, scenes, entry):
    key, spec, call = ENTRIES[entry]
    s = scenes[key]
    for name, (_, required, _) in spec.items():
        if not required:
            continue
        a = arrays(spec, N)
        a[name] = None
        rc = call(b2ctx.L, s.h, N, a)
        assert rc == B2_ERR_INVALID, (entry, name)
        assert entry in b2ctx.err(), (entry, name, b2ctx.err())


@pytest.mark.parametrize("entry", sorted(BAD))
def test_bad_id_is_refused(b2ctx, scenes, entry):
    key, spec, call = ENTRIES[entry]
    for kw, message in BAD[entry]:
        a = arrays(spec, N)
        for v in a.values():
            v.fill(SENTINEL)
        refused(b2ctx, call(b2ctx.L, scenes[key].h, N, a, **kw), message)
        for name, v in a.items():
            assert (v == SENTINEL).all(), name


@pytest.mark.parametrize("entry", sorted(ENTRIES))
def test_zero_items_succeed_and_write_nothing(b2ctx, scenes, entry):
    key, spec, call = ENTRIES[entry]
    a = arrays(spec, 0)
    for v in a.values():
        v.fill(SENTINEL)
    assert call(b2ctx.L, scenes[key].h, 0, a) == B2_OK, b2ctx.err()
    for name, v in a.items():
        assert (v == SENTINEL).all(), name


def test_optional_arrays_stay_optional(b2ctx, scenes):
    L = b2ctx.L
    rays = _rays(N)
    prim = np.zeros(N, np.float32)
    assert L.b2_trace(scenes["cornell"].h, C.c_uint64(N), _p(rays), C.c_int(0), C.c_int(1), None, None, None, _p(prim), None) == B2_OK
    assert L.b2_trace(scenes["cornell"].h, C.c_uint64(N), _p(rays), C.c_int(1), C.c_int(1), None, None, None, None, None) == B2_OK
    uv, out = _uv(N), np.zeros((N, 3), np.float32)
    assert L.b2_texture_eval(scenes["textured"].h, C.c_int(0), C.c_uint64(N), _p(uv), None, C.c_int(1), _p(out)) == B2_OK
    assert out.any()


def test_splat_refusals_and_zero_items(b2ctx):
    L = b2ctx.L
    pos, val = np.full((N, 2), 0.5, np.float32), np.ones((N, 4), np.float32)
    film = np.full((4, 4, 5), SENTINEL, np.float32)

    def splat(n, p, v, f):
        return L.b2_splat(b2ctx.h, C.c_int(4), C.c_int(4), C.c_int(0), C.c_float(0.5), C.c_uint64(n), _p(p), _p(v), _p(f))

    for args in ((None, val, film), (pos, None, film), (pos, val, None)):
        refused(b2ctx, splat(N, *args), "b2_splat")
    assert (film == SENTINEL).all()
    assert splat(0, pos, val, film) == B2_OK, b2ctx.err()
    assert not film.any()  # no samples: an empty film
