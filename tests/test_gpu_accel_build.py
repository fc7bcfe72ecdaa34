"""The device-side BVH build against the host builder: the same SceneDesc committed with accel_build="host" and "device" must give
byte-identical binary and 8-wide node arrays and the same leaf order (below an object-median split: the same set of triangles in every
binary leaf), hence bit-identical ray queries; device-built scenes pass the image-parity checks against the oracle."""
import os

import numpy as np
import pytest

from mitsuba_b200 import api
from mitsuba_b200.scene import (Bsdf, Camera, Instance, Mesh, RenderParams, SceneDesc, cornell_box, cube_mesh, look_at, material_ball,
                                stress_scene, uv_sphere)
from oracle import oracle_api as O

pytestmark = pytest.mark.gpu
REL_L2_TOL = 1e-3   # BASELINE.json north_star
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def rel_l2(a, b):
    return float(np.sqrt(((a.astype(np.float64) - b) ** 2).sum() / (b.astype(np.float64) ** 2).sum()))


def _cam():
    return Camera(look_at((0, 0, -4), (0, 0, 0), (0, 1, 0)), width=16, height=16)


def _soup(lo, hi):
    """One triangle per box whose own box is exactly [lo, hi]."""
    n = len(lo)
    P = np.empty((3 * n, 3), np.float32)
    P[0::3] = lo
    P[1::3] = np.stack([hi[:, 0], lo[:, 1], hi[:, 2]], 1)
    P[2::3] = np.stack([lo[:, 0], hi[:, 1], hi[:, 2]], 1)
    return SceneDesc([Mesh(P, np.arange(3 * n, dtype=np.uint32).reshape(-1, 3), bsdf=Bsdf("diffuse"))], _cam())


def _random_tris(n, seed, scale=1.0):
    rng = np.random.default_rng(seed)
    c = rng.uniform(-scale, scale, (n, 1, 3))
    P = (c + rng.normal(0, 0.02 * scale, (n, 3, 3))).astype(np.float32).reshape(-1, 3)
    return SceneDesc([Mesh(P, np.arange(3 * n, dtype=np.uint32).reshape(-1, 3), bsdf=Bsdf("diffuse"))], _cam())


def _invariance_soup(n=20000, seed=3):
    """The boxes of b2_bvh_thread_invariance (clustered sizes, an exact duplicate every 97th box), as triangles."""
    st = (seed * 747796405 + 2891336453) & 0xFFFFFFFF

    def rnd():
        nonlocal st
        st = (st * 747796405 + 2891336453) & 0xFFFFFFFF
        w = (((st >> ((st >> 28) + 4)) ^ st) * 277803737) & 0xFFFFFFFF
        return np.float32(((w >> 22) ^ w) >> 8) * np.float32(1.0 / 16777216.0)

    lo = np.zeros((n, 3), np.float32); hi = np.zeros((n, 3), np.float32)
    for i in range(n):
        c = (rnd() * np.float32(100) - np.float32(50), rnd() * np.float32(100) - np.float32(50), rnd() * np.float32(10) - np.float32(5))
        r = np.float32(0.01) + np.float32(0.3) * rnd() * rnd()
        if i > 0 and i % 97 == 0:
            lo[i], hi[i] = lo[i - 1], hi[i - 1]
            continue
        for a in range(3):
            lo[i, a] = c[a] - r * rnd(); hi[i, a] = c[a] + r * rnd()
    return _soup(lo, hi)


def _signed_zeros(n=3000, seed=5):
    """Every box touches 0 on every axis, with +0 and -0 both present as coordinates."""
    rng = np.random.default_rng(seed)
    P = rng.uniform(0.01, 1, (n, 3, 3)).astype(np.float32)
    for a in range(3):
        P[:, 1:, a] *= np.where(rng.random(n) < 0.5, 1, -1).astype(np.float32)[:, None]   # both other corners on one side of 0
        P[:, 0, a] = np.where(rng.random(n) < 0.5, np.float32(0.0), np.float32(-0.0))
    return SceneDesc([Mesh(P.reshape(-1, 3), np.arange(3 * n, dtype=np.uint32).reshape(-1, 3), bsdf=Bsdf("diffuse"))], _cam())


def _coincident(n=300, seed=6):
    """Boxes symmetric about the origin: every centroid is exactly 0, so every split is the object median."""
    rng = np.random.default_rng(seed)
    a = rng.uniform(0.1, 1, (n, 3)).astype(np.float32)
    s = rng.uniform(-1, 1, (n, 3)).astype(np.float32)
    P = np.stack([-a, a, a * s], 1)
    return SceneDesc([Mesh(P.reshape(-1, 3), np.arange(3 * n, dtype=np.uint32).reshape(-1, 3), bsdf=Bsdf("diffuse"))], _cam())


def _chain(n=300):
    """Tiny triangles at geometrically growing distances (up to 1.25^299 ~ 1e29, finite): SAH peels one off per level until the depth
    cap forces medians."""
    x = (1.25 ** np.arange(n)).astype(np.float32)
    s = x * np.float32(1e-4)
    P = np.zeros((n, 3, 3), np.float32)
    P[:, 0, 0] = x; P[:, 1, 0] = x + s; P[:, 2, 0] = x
    P[:, 1, 1] = s; P[:, 2, 2] = s
    return SceneDesc([Mesh(P.reshape(-1, 3), np.arange(3 * n, dtype=np.uint32).reshape(-1, 3), bsdf=Bsdf("diffuse"))], _cam())


def _instanced_two_groups():
    d = stress_scene(6, 24, 24, 64, 64, instanced=True)
    P, N, UV, I = uv_sphere((0, 0, 0), 0.6, 12, 24, with_uv=True)
    d.meshes.append(Mesh(P, I, N=N, UV=UV, bsdf=Bsdf("diffuse", reflectance=(0.6, 0.3, 0.2)), group=1))
    Pc, Ic = cube_mesh((-0.4, -0.9, -0.4), (0.4, -0.6, 0.4))
    d.meshes.append(Mesh(Pc, Ic, bsdf=Bsdf("diffuse", reflectance=(0.2, 0.6, 0.3)), group=2))
    for g, t in ((1, (0.5, 2.6, -1.0)), (1, (-2.0, 2.2, 0.5)), (2, (1.5, 1.0, 0.0))):
        M = np.eye(4); M[:3, 3] = t
        d.instances.append(Instance(g, M.astype(np.float32)))
    return d


def _sphere18k():
    P, N, UV, I = uv_sphere((0.3, -0.2, 0.1), 1.0, 96, 96, with_uv=True)
    return SceneDesc([Mesh(P, I, N=N, UV=UV, bsdf=Bsdf("diffuse"))], _cam())


# name -> (scene, whether the host builder takes object-median splits there)
CASES = {
    "tri65": (lambda: _random_tris(65, 1), False),
    "sphere18k": (_sphere18k, False),
    "invariance_soup": (_invariance_soup, False),
    "random300k": (lambda: _random_tris(300000, 2, 10.0), False),
    "signed_zeros": (_signed_zeros, False),
    "coincident": (_coincident, True),
    "depth_cap_chain": (_chain, True),
    "instanced": (_instanced_two_groups, False),
    "stress25": (lambda: stress_scene(25, width=64, height=64), False),
}


def _binary_leaves(nodes, n_leaf):
    """(start, count) of every binary leaf referenced by a node array without a top-level tree."""
    if not nodes:
        return [(0, n_leaf)]
    refs = np.frombuffer(nodes, np.int32).reshape(-1, 16)[:, 12:14].ravel()
    bits = ~refs[refs < 0].astype(np.int64) & 0xFFFFFFFF
    return list(zip((bits & 0x0FFFFFFF).tolist(), (bits >> 28).tolist()))


def _random_rays(d, n, seed):
    """Rays aimed at (near) the world triangles from around them; the distances scale with the target's own magnitude, so the
    geometric chain (coordinates up to 1e29) is hit as well."""
    P = np.concatenate([np.asarray(m.P, np.float64).reshape(-1, 3) for m in d.meshes if m.group < 0] or [np.zeros((1, 3))])
    span = P.max(0) - P.min(0)
    if d.instances:
        span = np.maximum(span, 8.0)
    rng = np.random.default_rng(seed)
    t = P[rng.integers(0, len(P), n)]
    scale = np.minimum(span.max(), 20 * np.abs(t).max(1, keepdims=True) + 1e-3)
    t = t + rng.normal(0, 1, (n, 3)) * 2.5e-3 * scale * np.where(scale < span.max(), 0.002, 1.0)
    o = t + rng.normal(0, 1, (n, 3)) * rng.uniform(0.05, 1.0, (n, 1)) * scale
    dirs = (t - o) / np.linalg.norm(t - o, axis=1, keepdims=True)
    maxt = np.where(rng.random(n) < 0.5, np.inf, rng.uniform(0, 2, n) * np.linalg.norm(t - o, axis=1))
    return np.concatenate([o, np.full((n, 1), 1e-4), dirs, maxt[:, None]], 1).astype(np.float32)


@pytest.fixture(scope="module", params=sorted(CASES))
def built(request, b2ctx):
    make, median = CASES[request.param]
    d = make()
    h = api.Scene(b2ctx, d, accel_build="host")
    g = api.Scene(b2ctx, d, accel_build="device")
    yield request.param, d, median, h, g
    h.close(); g.close()


def test_device_build_matches_host_build(built):
    name, d, median, h, g = built
    sh, sg = h.stats(), g.stats()
    assert sh["accel_build_mode"] == 0 and sg["accel_build_mode"] == 1
    for k in ("n_triangles", "n_bvh_nodes", "bvh_node_bytes"):   # includes whether the wide tree was dropped for depth
        assert sh[k] == sg[k], (name, k)
    a, b = h.accel_arrays(), g.accel_arrays()
    assert len(a["nodes"]) == len(b["nodes"]) and a["nodes"] == b["nodes"], name
    assert len(a["nodes8"]) == len(b["nodes8"]) and a["nodes8"] == b["nodes8"], name
    la, lb = a["leaf_prims"], b["leaf_prims"]
    assert len(la) == len(lb) == (d.n_triangles() if not d.instances else len(la))
    if not median:
        assert np.array_equal(la, lb), name
    else:   # the order inside a leaf below a median split is unspecified for the host builder
        leaves = _binary_leaves(a["nodes"], len(la))
        assert sum(c for _, c in leaves) == len(la)
        for s, c in leaves:
            assert np.array_equal(np.sort(la[s:s + c]), np.sort(lb[s:s + c])), (name, s, c)
    if name != "tri65":   # 65 triangles: the smallest scene that gets a tree
        assert sg["accel_build_ms"] > 0 and sh["accel_build_ms"] > 0


@pytest.mark.parametrize("parity", [True, False])
def test_ray_queries_bit_identical(built, parity):
    name, d, _, h, g = built
    rays = _random_rays(d, 100000, 11)
    for mode in (0, 1):
        th, uh, vh, ph = h.trace(rays, mode, parity=parity)
        tg, ug, vg, pg = g.trace(rays, mode, parity=parity)
        assert np.array_equal(ph, pg), (name, mode)
        for x, y in ((th, tg), (uh, ug), (vh, vg)):
            assert np.array_equal(x.view(np.uint32), y.view(np.uint32)), (name, mode)
    assert (ph != 0).mean() > 0.01, name   # occlusion: thousands of the rays do meet geometry


def _pair(ctx, d):
    g = api.Scene(ctx, d, accel_build="device")
    return g, O.OracleScene(d, sample_to_camera=g.sample_to_camera())


def test_device_built_cbox_image_parity(b2ctx):
    g, o = _pair(b2ctx, cornell_box(64, 64))
    rp = RenderParams(spp=32, sampler="sobol", rfilter="box")
    assert rel_l2(api.develop(g.render(rp, parity=True)[0]), O.develop(o.render(rp)[0])) <= REL_L2_TOL


def test_device_built_material_ball_image_parity(b2ctx):
    g, o = _pair(b2ctx, material_ball(Bsdf("diffuse", reflectance=(0.5, 0.4, 0.3)), 64, 64, 48, 96))
    assert g.stats()["accel_build_mode"] == 1 and g.stats()["n_triangles"] > 64
    rp = RenderParams(spp=32, sampler="sobol", rfilter="gaussian")
    assert rel_l2(api.develop(g.render(rp, parity=True)[0]), O.develop(o.render(rp)[0])) <= REL_L2_TOL


def test_device_built_instanced_image_parity(b2ctx):
    g, o = _pair(b2ctx, _instanced_two_groups())
    rp = RenderParams(spp=16, sampler="sobol", rfilter="box")
    assert rel_l2(api.develop(g.render(rp, parity=True)[0]), O.develop(o.render(rp)[0])) <= REL_L2_TOL


def test_load_xml_through_the_context_default(b2ctx):
    path = os.path.join(ROOT, "scenes", "cbox.xml")
    try:
        sc, _ = b2ctx.load_xml(path, accel_build="device")
        assert sc.stats()["accel_build_mode"] == 1
        sc.close()
        sc, _ = b2ctx.load_xml(path, accel_build="host")
        assert sc.stats()["accel_build_mode"] == 0
        sc.close()
    finally:
        b2ctx.set_accel_build("host")


def test_accel_build_errors(b2ctx):
    L = b2ctx.L
    d = _random_tris(100, 9)
    with pytest.raises(api.B2Error, match="accel_build must be one of"):
        api.Scene(b2ctx, d, accel_build="gpu")
    import ctypes as C
    h = C.c_void_p()
    assert L.b2_scene_create(b2ctx.h, C.byref(h)) == 0
    try:
        assert L.b2_scene_set_accel_build(h, C.c_int(7)) == 1
        assert "unknown mode 7" in b2ctx.err()
    finally:
        L.b2_scene_destroy(h)
    assert L.b2_context_set_accel_build(b2ctx.h, C.c_int(-1)) == 1 and "unknown mode -1" in b2ctx.err()
    sc = api.Scene(b2ctx, d, accel_build="device")
    assert L.b2_scene_set_accel_build(sc.h, C.c_int(0)) == 1
    assert "already committed" in b2ctx.err()
    n = C.c_uint64(0)
    assert L.b2_scene_get_accel(sc.h, C.c_int(3), None, C.byref(n)) == 1 and "unknown array" in b2ctx.err()
    assert L.b2_scene_get_accel(sc.h, C.c_int(0), None, C.byref(n)) == 0 and n.value > 0
    small = C.c_uint64(n.value - 1)
    buf = (C.c_uint8 * n.value)()
    assert L.b2_scene_get_accel(sc.h, C.c_int(0), buf, C.byref(small)) == 1 and "too small" in b2ctx.err()
