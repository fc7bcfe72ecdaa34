"""Parity tests proper: the CUDA path, through the C-ABI, against the oracle on the same seeded inputs.
Integer/index outputs (prim ids, occlusion bits, Sobol' words, counters) are compared exactly; floating point
within tolerances written next to each assertion; images by per-pixel relative L2 <= 1e-3 (BASELINE.json)."""
import dataclasses

import zlib

import numpy as np
import pytest

from bsdf_configs import configs
from mitsuba_b200 import api
from mitsuba_b200.scene import Bsdf, Camera, Mesh, RenderParams, SceneDesc, cornell_box, look_at, material_ball, uv_sphere
from oracle import oracle_api as O

pytestmark = pytest.mark.gpu
REL_L2_TOL = 1e-3   # BASELINE.json north_star


def rel_l2(a, b):
    return float(np.sqrt(((a.astype(np.float64) - b) ** 2).sum() / (b.astype(np.float64) ** 2).sum()))


def random_rays(rng, n, lo, hi):
    o = rng.uniform(lo, hi, (n, 3)).astype(np.float32)
    d = rng.normal(size=(n, 3)).astype(np.float32)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return np.concatenate([o, np.full((n, 1), 1e-4, np.float32), d, np.full((n, 1), np.inf, np.float32)], 1).astype(np.float32)


def pair(ctx, d):
    """Device scene + oracle scene from the same description (camera matrix handed over as float32)."""
    g = api.Scene(ctx, d)
    return g, O.OracleScene(d, sample_to_camera=g.sample_to_camera())


@pytest.fixture(scope="module")
def cbox(b2ctx):
    d = cornell_box(96, 96)
    g, o = pair(b2ctx, d)
    return d, g, o


def test_triaccel_records_bit_exact(cbox):
    _, g, o = cbox
    a, b = g.triaccel().view(np.uint32), o.triaccel().view(np.uint32)
    assert np.array_equal(a[:, :10], b[:, :10])   # words 10/11 hold ids with different meaning


def test_camera_rays_bit_exact(cbox):
    _, g, o = cbox
    assert np.allclose(g.sample_to_camera().ravel(), np.asarray(cornell_box(96, 96).camera.sample_to_camera()).ravel(), rtol=1e-6, atol=1e-6)
    pos = np.random.default_rng(1).uniform(0, 96, (5000, 2)).astype(np.float32)
    assert np.array_equal(g.camera_rays(pos, parity=True), o.camera_rays(pos))


def test_closest_hit_and_occlusion_exact(cbox):
    """Same TriAccel arithmetic, -fmad=false: (prim, t, u, v) must be bit identical to the kd-tree oracle."""
    _, g, o = cbox
    rays = random_rays(np.random.default_rng(2), 50000, 5, 550)
    t0, u0, v0, p0 = o.trace(rays, 0)
    t1, u1, v1, p1 = g.trace(rays, 0, parity=True)
    assert np.array_equal(p0, p1) and np.array_equal(t0, t1) and np.array_equal(u0, u1) and np.array_equal(v0, v1)
    rays[:, 7] = np.random.default_rng(3).uniform(20, 700, len(rays))
    assert np.array_equal(o.trace(rays, 1)[3], g.trace(rays, 1, parity=True)[3])
    # FMA build (plane-form triangle test, paired flat-leaf records): same primitive, t within a few ulp -- except rays that graze an
    # edge shared by two triangles, where either neighbour is a correct answer
    rays[:, 7] = np.inf
    t2, u2, v2, p2 = g.trace(rays, 0, parity=False)
    same = p2 == p0
    assert same.mean() > 0.9995, same.mean()
    hit = same & (p0 != 0xFFFFFFFF)
    # scene scale 550: __fdividef + FMA contraction, cancellation in d0 - N.o
    assert np.allclose(t2[hit], t0[hit], rtol=1e-4, atol=2e-2)
    assert np.allclose(u2[hit], u0[hit], atol=2e-4) and np.allclose(v2[hit], v0[hit], atol=2e-4)
    assert np.array_equal(p2 == 0xFFFFFFFF, p0 == 0xFFFFFFFF) or (np.not_equal(p2 == 0xFFFFFFFF, p0 == 0xFFFFFFFF)).mean() < 2e-4


def test_traversal_large_mesh_exact(b2ctx):
    """BVH (device) vs kd-tree (oracle) on an 18k-triangle mesh, incl. rays starting on the surface (adaptive epsilon)."""
    P, N, UV, I = uv_sphere((0.3, -0.2, 0.1), 1.0, 96, 96, with_uv=True)
    d = SceneDesc([Mesh(P, I, N=N, UV=UV, bsdf=Bsdf("diffuse"))], Camera(look_at((0, 0, -4), (0, 0, 0), (0, 1, 0)), width=16, height=16))
    g, o = pair(b2ctx, d)
    rng = np.random.default_rng(4)
    rays = random_rays(rng, 40000, -2, 2)
    surf = P[rng.integers(0, len(P), 10000)]
    rays[:10000, :3] = surf
    a, b = o.trace(rays, 0), g.trace(rays, 0, parity=True)
    assert np.array_equal(a[3], b[3]) and np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])
    assert (a[3] != 0xFFFFFFFF).mean() > 0.15


@pytest.mark.parametrize("kind,seed", [("sobol", 0), ("sobol", 12345), ("independent", 0), ("independent", 99)])
def test_sampler_streams_exact(cbox, kind, seed):
    """Sampler state in registers: the first 24 dimensions of (pixel, sample) are the same 32-bit words."""
    _, g, o = cbox
    for (px, py, s) in [(0, 0, 0), (1, 0, 1), (5, 77, 3), (95, 95, 15), (40, 2, 1000)]:
        assert np.array_equal(g.sampler_stream(kind, seed, 1024, px, py, s, 24), o.sampler_stream(kind, seed, 1024, px, py, s, 24))


@pytest.mark.parametrize("name", sorted(configs()))
def test_bsdf_eval_sample_parity(b2ctx, name):
    """BSDF::eval / pdf / sample on the device vs the oracle for the reference's fixture parameters.
    Tolerance 2e-4 relative (CUDA libm transcendentals are within 1-2 ulp of glibc; a handful of inputs land on
    opposite sides of a branch -- those are counted and bounded instead)."""
    b = configs()[name]
    d = cornell_box(16, 16)
    d.meshes[0].bsdf = b
    g = api.Scene(b2ctx, d)
    flat, ids = d.flat_bsdfs()
    mid = ids[0]
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    n = 20000

    def sph(n):
        v = rng.normal(size=(n, 3)).astype(np.float32)
        return v / np.linalg.norm(v, axis=1, keepdims=True)
    wi, wo = sph(n), sph(n)
    f0, p0 = O.bsdf_eval(flat, mid, wi, wo)
    f1, p1 = g.bsdf_eval(mid, wi, wo, parity=True)
    assert np.allclose(f1, f0, rtol=2e-4, atol=1e-6) and np.allclose(p1, p0, rtol=2e-4, atol=1e-6)
    s = rng.uniform(size=(n, 3)).astype(np.float32)
    r0, r1 = O.bsdf_sample(flat, mid, wi, s), g.bsdf_sample(mid, wi, s, parity=True)
    same = (r0["type"] == r1["type"]) & ((np.abs(r0["weight"]).sum(1) > 0) == (np.abs(r1["weight"]).sum(1) > 0))
    assert same.mean() > 0.999
    ok = same & (np.abs(r0["weight"]).sum(1) > 0)
    close = np.isclose(r1["wo"][ok], r0["wo"][ok], rtol=0, atol=5e-4).all(1) & np.isclose(r1["pdf"][ok], r0["pdf"][ok], rtol=5e-3, atol=1e-5) & \
        np.isclose(r1["weight"][ok], r0["weight"][ok], rtol=5e-3, atol=1e-5).all(1)
    assert close.mean() > 0.998, (name, close.mean())
    assert np.array_equal(r0["eta"][ok], r1["eta"][ok])


def test_emitter_direct_sampling_parity(cbox):
    _, g, o = cbox
    rng = np.random.default_rng(5)
    ref = np.concatenate([rng.uniform(50, 500, (8000, 3)) * [1, 0.6, 1], np.zeros((8000, 3))], 1).astype(np.float32)
    ref[::2, 3:] = [0, 1, 0]
    s = rng.uniform(size=(8000, 2)).astype(np.float32)
    a, b = o.sample_emitter_direct(ref, s), g.sample_emitter_direct(ref, s, parity=True)
    assert np.array_equal(a[:, 8], b[:, 8])                       # visibility bits
    vis = a[:, 8] == 1
    assert np.array_equal(a[vis], b[vis])                          # -fmad=false: bit identical


@pytest.mark.parametrize("kind,param", [("box", 0.5), ("gaussian", 0.5), ("gaussian", 0.8)])
def test_film_put_parity(b2ctx, kind, param):
    """ImageBlock::put: atomics change the summation order only."""
    rng = np.random.default_rng(6)
    W, H, n = 150, 77, 30000
    pos = rng.uniform(0, [W, H], (n, 2)).astype(np.float32)
    pos[:200] = np.floor(pos[:200])
    val = rng.uniform(0, 2, (n, 4)).astype(np.float32)
    a, b = O.splat(W, H, kind, param, pos, val), b2ctx.splat(W, H, kind, param, pos, val)
    assert np.allclose(a, b, rtol=2e-5, atol=2e-5)
    assert np.array_equal(a[..., 4] > 0, b[..., 4] > 0)


@pytest.mark.parametrize("rfilter", ["box", "gaussian"])
@pytest.mark.parametrize("parity", [True, False])
def test_cornell_image_parity(cbox, rfilter, parity):
    """Config 1 class: Cornell box, sobol, both filters; relative L2 of the developed image vs the oracle."""
    _, g, o = cbox
    rp = RenderParams(spp=32, sampler="sobol", rfilter=rfilter)
    fo, so = o.render(rp)
    fg, sg = g.render(rp, parity=parity)
    e = rel_l2(api.develop(fg), O.develop(fo))
    assert e <= REL_L2_TOL, e
    if parity:
        # -fmad=false: the only differences left are CUDA-vs-glibc sincosf (1 ulp), which flip a handful of paths
        assert e < 2e-4
        # the three statistics of the reference (path.cpp:24, skdtree.cpp:46-47)
        assert sg["samples"] == so["samples"] and sg["bad_samples"] == 0
        for a, b in ((sg["rays"], so["rays"]), (sg["shadow_rays"], so["shadowRays"]), (sg["path_length_sum"], so["pathLengthSum"])):
            assert abs(a - b) <= 1e-4 * b
    assert np.allclose(fg[..., 4], fo[..., 4], rtol=1e-5, atol=1e-5)


def test_independent_sampler_image_parity(cbox):
    _, g, o = cbox
    rp = RenderParams(spp=16, sampler="independent", seed=7, rfilter="box")
    fo, _ = o.render(rp)
    fg, _ = g.render(rp, parity=True)
    assert rel_l2(api.develop(fg), O.develop(fo)) < 2e-4


@pytest.mark.parametrize("kw", [dict(max_depth=1), dict(max_depth=2), dict(max_depth=4, rr_depth=2), dict(strict_normals=True), dict(hide_emitters=True),
                                dict(seed=4711)])
def test_integrator_properties_parity(cbox, kw):
    _, g, o = cbox
    rp = RenderParams(spp=16, sampler="sobol", rfilter="box", **kw)
    fo, so = o.render(rp)
    fg, sg = g.render(rp, parity=True)
    # (with hideEmitters the bright light pixels leave the denominator, so the same handful of flipped paths weighs ~10x more)
    assert rel_l2(api.develop(fg), O.develop(fo)) < (REL_L2_TOL if kw.get("hide_emitters") else 2e-4)
    assert abs(sg["path_length_sum"] - so["pathLengthSum"]) <= 1e-4 * so["pathLengthSum"] + 2 and abs(sg["rays"] - so["rays"]) <= 1e-4 * so["rays"] + 2


MATERIALS = {
    "roughconductor_ggx": Bsdf("roughconductor", distribution="ggx", alpha_u=0.1, alpha_v=0.1, eta=(0.2004, 0.9240, 1.1022), k=(3.9129, 2.4528, 2.1421)),
    "roughconductor_beckmann_aniso": Bsdf("roughconductor", distribution="beckmann", alpha_u=0.05, alpha_v=0.3, eta=(0.2004, 0.9240, 1.1022), k=(3.9129, 2.4528, 2.1421)),
    "roughdielectric_ggx": Bsdf("roughdielectric", distribution="ggx", alpha_u=0.1, alpha_v=0.1, int_ior="bk7", ext_ior="air"),
    "roughdielectric_beckmann": Bsdf("roughdielectric", distribution="beckmann", alpha_u=0.3, alpha_v=0.3, int_ior=1.5, ext_ior=1.0),
    "coating_roughconductor": Bsdf("coating", int_ior=1.5, ext_ior=1.0, nested=Bsdf("roughconductor", distribution="ggx", alpha_u=0.2, alpha_v=0.2,
                                                                                   eta=(0.2004, 0.9240, 1.1022), k=(3.9129, 2.4528, 2.1421))),
    "coating_diffuse_absorbing": Bsdf("coating", int_ior=1.5, ext_ior=1.0, sigma_a=(0.1, 0.2, 0.3), thickness=2.0, nested=Bsdf("diffuse", reflectance=(0.7, 0.6, 0.5))),
}


@pytest.mark.parametrize("name", sorted(MATERIALS))
@pytest.mark.parametrize("sorted_shading", [True, False])
def test_material_ball_image_parity(b2ctx, name, sorted_shading):
    """Config 3 class (reduced size): material ball with smooth vertex normals; material-sorted and unsorted dispatch."""
    d = material_ball(MATERIALS[name], 64, 64, 48, 96)
    g, o = pair(b2ctx, d)
    rp = RenderParams(spp=32, sampler="sobol", rfilter="gaussian")
    fo, so = o.render(rp)
    fg, sg = g.render(rp, parity=True, flags=0 if sorted_shading else 2)
    e = rel_l2(api.develop(fg), O.develop(fo))
    assert e <= REL_L2_TOL, (name, e)
    assert abs(sg["path_length_sum"] - so["pathLengthSum"]) <= 1e-3 * so["pathLengthSum"]
    if not sorted_shading:
        return
    # Throughput build (the one bench.py times).  An ulp-level difference flips a fraction f of the paths (of order 1e-5; most for a rough
    # dielectric, fewest for diffuse); a flipped path is an unrelated sample of a heavy-tailed estimator, so the image error behaves like
    # 3.7 * sqrt(f / spp), which at low sample counts exceeds 1e-3 whatever the kernel does.  The 1e-3 bar is
    # therefore tested where it is resolvable, together with the diagnostic itself (fraction of pixels whose path lengths changed).
    # (flags 256 forces the throughput kernels: by default a `path` render of a scene with a transmissive BSDF is dispatched to the IEEE
    # kernels for exactly this reason, which the last assertion checks)
    rp_hi = RenderParams(spp=2048, sampler="sobol", rfilter="gaussian")
    fo_hi, so_hi = o.render(rp_hi)
    fg_hi, sg_hi = g.render(rp_hi, parity=False, flags=256)
    assert rel_l2(api.develop(fg_hi), O.develop(fo_hi)) <= REL_L2_TOL, name
    assert abs(sg_hi["path_length_sum"] - so_hi["pathLengthSum"]) <= 2e-4 * so_hi["pathLengthSum"]
    g.render(rp, parity=True, flags=32); pp = g.pixel_stats()
    g.render(rp, parity=False, flags=32 | 256); pf = g.pixel_stats()
    assert (pp != pf).sum() <= 2e-4 * 64 * 64 * 32, (name, int((pp != pf).sum()))   # <= 2e-4 of the paths change length (measured <= 5e-5)
    if "dielectric" in name:
        g.render(rp, parity=False, flags=32)
        assert np.array_equal(g.pixel_stats(), pp)   # default dispatch of a transmissive scene = the IEEE kernels


MATERIALS_F3 = {   # SURVEY.md 8f-3 plugins (generic shading kernel)
    "dielectric": Bsdf("dielectric", int_ior="bk7", ext_ior="air"),
    "conductor": Bsdf("conductor", eta=(0.2004, 0.9240, 1.1022), k=(3.9129, 2.4528, 2.1421)),
    "plastic": Bsdf("plastic", diffuse_reflectance=(0.1, 0.27, 0.36)),
    "plastic_nonlinear": Bsdf("plastic", diffuse_reflectance=(0.6, 0.3, 0.2), nonlinear=True, int_ior=1.9),
    "twosided_plastic": Bsdf("twosided", nested=Bsdf("plastic", diffuse_reflectance=(0.5, 0.2, 0.2)), nested_back=Bsdf("diffuse", reflectance=(0.1, 0.6, 0.1))),
}


@pytest.mark.parametrize("name", sorted(MATERIALS_F3))
def test_f3_material_ball_image_parity(b2ctx, name):
    d = material_ball(MATERIALS_F3[name], 64, 64, 48, 96)
    # the ground becomes a two-sided diffuse sheet seen from below by part of the light transport
    d.meshes[0].bsdf = Bsdf("twosided", nested=Bsdf("diffuse", reflectance=(0.5, 0.5, 0.5)))
    g, o = pair(b2ctx, d)
    rp = RenderParams(spp=32, sampler="sobol", rfilter="gaussian")
    fo, so = o.render(rp)
    fg, sg = g.render(rp, parity=True)
    e = rel_l2(api.develop(fg), O.develop(fo))
    assert e <= REL_L2_TOL, (name, e)
    assert abs(sg["path_length_sum"] - so["pathLengthSum"]) <= 1e-3 * so["pathLengthSum"]
    fg2, _ = g.render(rp, parity=False)
    assert rel_l2(api.develop(fg2), O.develop(fo)) <= REL_L2_TOL


def test_twosided_sheet_is_lit_from_both_sides(b2ctx):
    """A one-sided diffuse sheet is black from behind (diffuse.cpp:112-113); wrapped in `twosided` it is not."""
    from mitsuba_b200.scene import _quad
    def scene(bsdf):
        P, I = _quad([(-1, 0, -1), (-1, 0, 1), (1, 0, 1), (1, 0, -1)], (0, 1, 0))
        sheet = Mesh(P, I, bsdf=bsdf)
        P, I = _quad([(-0.5, -2, -0.5), (-0.5, -2, 0.5), (0.5, -2, 0.5), (0.5, -2, -0.5)], (0, 1, 0))
        light = Mesh(P, I, bsdf=Bsdf("diffuse", reflectance=(0, 0, 0)), radiance=(10, 10, 10))
        return SceneDesc([sheet, light], Camera(look_at((0, -1.5, -3), (0, 0, 0), (0, 1, 0)), fov=40, width=32, height=32))
    rp = RenderParams(spp=16, sampler="sobol", rfilter="box")
    one, _ = api.Scene(b2ctx, scene(Bsdf("diffuse"))).render(rp, parity=True)
    two_d = scene(Bsdf("twosided", nested=Bsdf("diffuse")))
    g, o = pair(b2ctx, two_d)
    two, _ = g.render(rp, parity=True)
    fo, _ = o.render(rp)
    centre = (slice(12, 20), slice(12, 20))
    assert api.develop(one)[centre].max() == 0 and api.develop(two)[centre].mean() > 0.05
    assert rel_l2(api.develop(two), O.develop(fo)) < 2e-4


def test_invalid_nesting_is_rejected(b2ctx):
    d = cornell_box(16, 16)
    d.meshes[0].bsdf = Bsdf("twosided", nested=Bsdf("dielectric"))
    with pytest.raises(api.B2Error, match="without a transmission component"):   # twosided.cpp:105-107
        api.Scene(b2ctx, d)


@pytest.mark.parametrize("mat", ["diffuse", "roughdielectric", "plastic"])
def test_constant_environment_emitter_parity(b2ctx, mat):
    """`constant` emitter (src/emitters/constant.cpp): environment hit by BSDF sampling (MIS with the cosine / uniform-sphere
    direct-sampling density), direct sampling through the scene bounding sphere, hideEmitters, together with an area light."""
    b = {"diffuse": Bsdf("diffuse", reflectance=(0.6, 0.5, 0.4)), "roughdielectric": MATERIALS["roughdielectric_ggx"], "plastic": MATERIALS_F3["plastic"]}[mat]
    d = material_ball(b, 64, 64, 32, 64)
    d.meshes = [m for m in d.meshes if m.name != "backdrop"]
    d.env_radiance = (0.4, 0.6, 1.0); d.env_sampling_weight = 2.0
    g, o = pair(b2ctx, d)
    # glossy transmission: one libm-flipped path costs ~1e-3 at 32 spp on 64 x 64 pixels (heavy-tailed estimator), so it runs at 512 spp
    spp = 512 if mat == "roughdielectric" else 32
    for kw in (dict(), dict(hide_emitters=True), dict(max_depth=2)):
        rp = RenderParams(spp=spp, sampler="sobol", rfilter="box", **kw)
        fo, so = o.render(rp)
        fg, sg = g.render(rp, parity=True)
        assert rel_l2(api.develop(fg), O.develop(fo)) <= 3e-4, (mat, kw)
        assert abs(sg["path_length_sum"] - so["pathLengthSum"]) <= 1e-3 * so["pathLengthSum"]
    fg2, _ = g.render(RenderParams(spp=2048, sampler="sobol", rfilter="box"), parity=False)
    fo, _ = o.render(RenderParams(spp=2048, sampler="sobol", rfilter="box"))
    assert rel_l2(api.develop(fg2), O.develop(fo)) <= REL_L2_TOL


def test_environment_only_scene_and_errors(b2ctx):
    P, N, _, I = uv_sphere((0, 0, 0), 1.0, 24, 48)
    d = SceneDesc([Mesh(P, I, N=N, bsdf=Bsdf("diffuse", reflectance=(1, 1, 1)))], Camera(look_at((0, 0, -4), (0, 0, 0), (0, 1, 0)), fov=40, width=32, height=32),
                  env_radiance=(0.7, 0.8, 0.9))
    g, o = pair(b2ctx, d)
    rp = RenderParams(spp=64, sampler="independent", rfilter="box", rr_depth=50)
    fg, _ = g.render(rp, parity=False)
    assert np.allclose(api.develop(fg).reshape(-1, 3).mean(0), (0.7, 0.8, 0.9), rtol=3e-3)   # white furnace
    fo, _ = o.render(rp)
    fg, _ = g.render(rp, parity=True)
    assert rel_l2(api.develop(fg), O.develop(fo)) <= 3e-4
    # volpath treats the environment the same way when there is no medium
    fv, _ = g.render(dataclasses.replace(rp, integrator="volpath"), parity=True)
    fov, _ = o.render(dataclasses.replace(rp, integrator="volpath"))
    assert rel_l2(api.develop(fv), O.develop(fov)) <= 3e-4


def test_uv_tangent_frames_parity(b2ctx):
    """Meshes with texcoords take the UV-tangent shading frame (trimesh.cpp:683-735, skdtree.h:373-380): anisotropic BSDF."""
    P, N, UV, I = uv_sphere((0, 1, 0), 1.0, 32, 64, with_uv=True)
    d = material_ball(MATERIALS["roughconductor_beckmann_aniso"], 48, 48, 8, 8)
    d.meshes[1] = Mesh(P, I, N=N, UV=UV, bsdf=MATERIALS["roughconductor_beckmann_aniso"])
    g, o = pair(b2ctx, d)
    rp = RenderParams(spp=32, sampler="sobol", rfilter="box")
    fo, _ = o.render(rp); fg, _ = g.render(rp, parity=True)
    assert rel_l2(api.develop(fg), O.develop(fo)) <= REL_L2_TOL


def test_sample_range_shards_add_up(cbox):
    """Multi-GPU sharding property on one device: films of disjoint sample ranges add up to the full film."""
    _, g, _ = cbox
    rp = RenderParams(spp=32, sampler="sobol", rfilter="gaussian")
    full, _ = g.render(rp, parity=True)
    parts = [g.render(dataclasses.replace(rp, sample_lo=a, sample_hi=b), parity=True)[0] for a, b in ((0, 8), (8, 16), (16, 32))]
    s = parts[0] + parts[1] + parts[2]
    assert np.allclose(s, full, rtol=2e-5, atol=2e-5)


def test_pool_size_independence(cbox):
    """The wavefront pool size only changes scheduling: same film up to atomic summation order."""
    _, g, _ = cbox
    rp = RenderParams(spp=16, sampler="sobol", rfilter="box")
    a, sa = g.render(rp, parity=True, pool_size=4096)
    b, sb = g.render(rp, parity=True, pool_size=1 << 20)
    assert np.allclose(a, b, rtol=2e-5, atol=2e-5)
    assert sa["rays"] == sb["rays"] and sa["path_length_sum"] == sb["path_length_sum"]


def test_full_size_properties(b2ctx):
    """BASELINE config 2 geometry (1024 x 1024), reduced spp: size-independent properties --
    (i) weight channel = spp * (filter norm)^2 + corner-sample spill exactly as the oracle's block logic predicts for the
        box filter: every pixel receives its own spp samples; (ii) radiance linearity: doubling L doubles RGB bit for bit;
    (iii) sample counters; (iv) no invalid samples."""
    d = cornell_box(1024, 1024)
    g = api.Scene(b2ctx, d)
    rp = RenderParams(spp=8, sampler="sobol", rfilter="box")
    f1, s1 = g.render(rp, parity=True)
    assert s1["samples"] == 1024 * 1024 * 8 and s1["bad_samples"] == 0 and s1["dim_overflow"] == 0
    tab, _, _ = O.filter_table("box", 0.5)
    w0 = np.float32(tab[0]) * np.float32(tab[0])
    # each pixel: 8 own samples (+ up to 3 corner samples of right/lower neighbours, box.cpp:41 radius epsilon)
    k = np.rint(f1[..., 4] / w0)
    assert np.allclose(f1[..., 4], k * w0, rtol=1e-5) and k.min() >= 8 and k.max() <= 11
    d2 = cornell_box(1024, 1024)
    d2.meshes[-1].radiance = tuple(2 * x for x in d2.meshes[-1].radiance)
    f2, s2 = api.Scene(b2ctx, d2).render(rp, parity=True)
    assert s2["rays"] == s1["rays"] and s2["path_length_sum"] == s1["path_length_sum"]
    rgb1, rgb2 = api.develop(f1), api.develop(f2)
    assert np.allclose(rgb2, 2 * rgb1, rtol=1e-5, atol=1e-7)
    # a 64x64 crop of the same scene rendered by the oracle at the same resolution is too slow; instead compare the
    # image against an independent-resolution invariant: mean radiance of the two renders agrees to MC noise
    assert abs(rgb1.mean() - 0.5 * rgb2.mean()) < 1e-5


def test_error_behaviour(b2ctx):
    """Same argument checks and messages as the reference constructors."""
    d = cornell_box(16, 16)
    g = api.Scene(b2ctx, d)
    with pytest.raises(api.B2Error, match="rrDepth"):
        g.render(RenderParams(spp=1, rr_depth=0))
    with pytest.raises(api.B2Error, match="maxDepth"):
        g.render(RenderParams(spp=1, max_depth=0))
    d.meshes[0].bsdf = Bsdf("roughdielectric", int_ior=1.5, ext_ior=1.5)
    with pytest.raises(api.B2Error, match="indices of refraction"):
        api.Scene(b2ctx, d)


def test_traversal_counters(b2ctx):
    """b2_trace_device in counting mode reports node visits / triangle tests (the E_trav, E_prim of the roofline model)."""
    import torch
    P, N, _, I = uv_sphere((0, 0, 0), 1.0, 64, 64)
    d = SceneDesc([Mesh(P, I, N=N, bsdf=Bsdf("diffuse"))], Camera(look_at((0, 0, -4), (0, 0, 0), (0, 1, 0)), width=16, height=16))
    g = api.Scene(b2ctx, d)
    n = 1 << 16
    rays = torch.tensor(random_rays(np.random.default_rng(11), n, -0.3, 0.3), device="cuda").contiguous()
    out = torch.zeros((n, 4), device="cuda")
    g.trace_device(rays, out, n, mode=0 | 2)
    st = g.stats()
    assert st["node_visits"] > 4 * n and st["prim_tests"] > n            # every ray starts inside the sphere and must hit it
    prim = out[:, 3].view(torch.int32)
    assert int((prim >= 0).sum()) == n


def test_ragged_film_small_pool_high_spp_terminates(b2ctx):
    """Film sizes that are not multiples of the 8x8 work tiles must not consume pool slots for pixels outside the film: with a 1024-slot
    pool, 20x12 pixels and 64 spp the old tile enumeration (3x2 tiles = 384 items per sample for 240 pixels) ran out of slots."""
    d = cornell_box(20, 12)
    g, o = pair(b2ctx, d)
    rp = RenderParams(spp=64, sampler="sobol", rfilter="box")
    fg, sg = g.render(rp, parity=True, pool_size=1024)
    fo, so = o.render(rp)
    assert sg["samples"] == 20 * 12 * 64 == so["samples"]
    assert np.allclose(fg[..., 4], fo[..., 4], rtol=1e-5, atol=1e-5)
    assert rel_l2(api.develop(fg), O.develop(fo)) < 5e-4
    # 100x100 @ 8 spp through a 4096-slot pool: 13x13 tiles used to waste 6900 of 16900 items per sample
    d = cornell_box(100, 100)
    g = api.Scene(b2ctx, d)
    f, st = g.render(RenderParams(spp=8, sampler="sobol", rfilter="box"), parity=False, pool_size=4096)
    assert st["samples"] == 100 * 100 * 8 and np.rint(f[..., 4]).min() >= 8


def test_open_scene_without_a_diffuse_class(b2ctx):
    """Material-sorted dispatch on a scene with two BSDF classes but no diffuse mesh, open to a constant environment: rays that leave the
    scene must still be retired (they are binned into the first class that has a shading kernel)."""
    d = material_ball(MATERIALS["roughdielectric_ggx"], 48, 48, 24, 48)
    d.meshes = [m for m in d.meshes if m.name in ("ground", "ball")]
    d.meshes[0].bsdf = MATERIALS["roughconductor_ggx"]
    d.env_radiance = (0.5, 0.6, 0.8)
    g, o = pair(b2ctx, d)
    rp = RenderParams(spp=16, sampler="sobol", rfilter="box")
    fo, so = o.render(rp)
    for flags in (0, 2):
        fg, sg = g.render(rp, parity=True, flags=flags)
        assert sg["samples"] == so["samples"]
        assert rel_l2(api.develop(fg), O.develop(fo)) <= REL_L2_TOL


def test_crop_window_parity(b2ctx):
    """Film crop window (film.cpp:36-47): the crop is the film the integrator sees; device vs oracle on the same camera matrix."""
    d = cornell_box(96, 64)
    d.camera = dataclasses.replace(d.camera, crop=(17, 9, 43, 33))
    g, o = pair(b2ctx, d)
    assert (g.W, g.H) == (43, 33)
    assert np.allclose(g.sample_to_camera(), d.camera.sample_to_camera(), rtol=1e-6, atol=1e-6)
    rp = RenderParams(spp=16, sampler="sobol", rfilter="gaussian")
    fo, so = o.render(rp); fg, sg = g.render(rp, parity=True)
    assert fg.shape == (33, 43, 5) and sg["samples"] == 43 * 33 * 16
    assert rel_l2(api.develop(fg), O.develop(fo)) < 5e-4
    with pytest.raises(api.B2Error, match="Invalid crop window"):
        bad = cornell_box(32, 32)
        bad.camera = dataclasses.replace(bad.camera, crop=(10, 10, 30, 8))
        api.Scene(b2ctx, bad)


def test_ragged_film_and_non_square(b2ctx):
    """Film sizes that are not multiples of the 8x8 work tiles / 32x32 render blocks, W != H (edge handling of the splat)."""
    d = cornell_box(70, 45)
    g, o = pair(b2ctx, d)
    for rf in ("box", "gaussian"):
        rp = RenderParams(spp=8, sampler="sobol", rfilter=rf)
        fo, so = o.render(rp); fg, sg = g.render(rp, parity=True)
        assert sg["samples"] == 70 * 45 * 8 == so["samples"]
        assert np.allclose(fg[..., 4], fo[..., 4], rtol=1e-5, atol=1e-5)
        assert rel_l2(api.develop(fg), O.develop(fo)) < 5e-4
    d1 = cornell_box(1, 1)
    g1, o1 = pair(b2ctx, d1)
    rp = RenderParams(spp=64, sampler="sobol", rfilter="box")
    f1, _ = g1.render(rp, parity=True); f0, _ = o1.render(rp)
    assert np.allclose(f1, f0, rtol=1e-3, atol=1e-4)


def test_sobol_indices_beyond_32_bits(b2ctx):
    """Config-5 class index range: 2048^2 film, sample indices >= 1024 -> 33-bit Sobol' indices (nibble tables past word 0)."""
    d = cornell_box(2048, 2048)
    g, o = pair(b2ctx, d)
    for (px, py, s) in [(0, 0, 2047), (2047, 2047, 2047), (1234, 77, 1500), (5, 2000, 1024)]:
        a, b = g.sampler_stream("sobol", 0, 2048, px, py, s, 16), o.sampler_stream("sobol", 0, 2048, px, py, s, 16)
        assert np.array_equal(a, b)
    idx = O.sobol_lookup(11, np.array([2047], np.uint32), 2047, 2047)[0]
    assert int(idx) >= 1 << 32


def test_degenerate_and_emitterless_scenes(b2ctx):
    """k = 3 TriAccel records (zero-area triangles, triaccel.h:75-78) are never hit; a scene without emitters renders black."""
    d = cornell_box(32, 32)
    m = d.meshes[0]
    m.P = np.concatenate([m.P, np.array([[100, 100, 100], [100, 100, 100], [200, 200, 200]], np.float32)])
    m.idx = np.concatenate([m.idx, np.array([[12, 13, 14]], np.uint32)])
    g, o = pair(b2ctx, d)
    rp = RenderParams(spp=8, sampler="sobol", rfilter="box")
    fo, _ = o.render(rp); fg, st = g.render(rp, parity=True)
    assert st["n_triangles"] == 33 and rel_l2(api.develop(fg), O.develop(fo)) < 5e-4
    d2 = cornell_box(32, 32)
    d2.meshes[-1].radiance = None
    g2 = api.Scene(b2ctx, d2)
    f2, s2 = g2.render(rp, parity=True)
    assert not f2[..., :3].any() and s2["samples"] == 32 * 32 * 8 and s2["shadow_rays"] == 0


def test_cancel_returns_status(b2ctx):
    """Integrator::cancel (integrator.h:90-93): a cancel issued from another thread stops the host loop with B2_ERR_CANCELLED."""
    import threading, time, ctypes as C
    d = cornell_box(512, 512)
    g = api.Scene(b2ctx, d)
    p = api.make_params(RenderParams(spp=4096, sampler="sobol", rfilter="box"), False, 0, False, 0)
    film = np.zeros((512, 512, 5), np.float32)
    rc = {}
    t = threading.Thread(target=lambda: rc.setdefault("rc", g.L.b2_render(g.h, C.byref(p), film.ctypes.data_as(C.POINTER(C.c_float)))))
    t.start(); time.sleep(0.05)
    t0 = time.time()
    while t.is_alive() and time.time() - t0 < 60:   # b2_render clears the flag when it starts: keep asking until it lands
        g.L.b2_cancel(g.h); time.sleep(0.005)
    t.join(timeout=60)
    assert not t.is_alive() and rc["rc"] == 5
    f, s = g.render(RenderParams(spp=2, sampler="sobol", rfilter="box"))       # the scene stays usable
    assert s["samples"] == 512 * 512 * 2


# ---- instancing (SURVEY.md 8f-2): src/shapes/{shapegroup,instance}.cpp ----
def _instanced_scene(n=5, res=48):
    from mitsuba_b200.scene import Instance, stress_scene
    d = stress_scene(n, 20, 20, res, res, instanced=True)
    # a second group with two meshes (one with UVs -> tangent frames through the instance transform), rotated + sheared instances
    P, N, UV, I = uv_sphere((0, 0, 0), 0.6, 12, 24, with_uv=True)
    # anisotropic, so the UV tangent frame matters, but not mirror-like: a near-specular lobe on a coarse sphere turns single
    # fast-math perturbations into isolated bright pixels that dominate the L2 of a 48x48 image
    aniso = Bsdf("roughconductor", distribution="beckmann", alpha_u=0.15, alpha_v=0.4, eta=(0.2004, 0.9240, 1.1022), k=(3.9129, 2.4528, 2.1421))
    d.meshes.append(Mesh(P, I, N=N, UV=UV, bsdf=aniso, group=1))
    from mitsuba_b200.scene import cube_mesh
    Pc, Ic = cube_mesh((-0.4, -0.9, -0.4), (0.4, -0.6, 0.4))
    d.meshes.append(Mesh(Pc, Ic, bsdf=Bsdf("diffuse", reflectance=(0.2, 0.6, 0.3)), group=1))
    c, s_ = np.cos(0.7), np.sin(0.7)
    M = np.eye(4); M[:3, :3] = np.array([[c, 0, s_], [0, 1, 0], [-s_, 0, c]]) @ np.diag([1.3, 0.8, 1.0]); M[0, 1] = 0.2; M[:3, 3] = (0.5, 2.6, -1.0)
    d.instances.append(Instance(1, M.astype(np.float32)))
    M2 = np.eye(4); M2[:3, :3] *= 0.7; M2[:3, 3] = (-2.0, 2.2, 0.5)
    d.instances.append(Instance(1, M2.astype(np.float32)))
    return d


def test_instanced_scene_image_parity(b2ctx):
    d = _instanced_scene()
    g, o = pair(b2ctx, d)
    st0 = g.stats()
    assert st0["n_triangles"] == d.n_triangles()
    for rp in (RenderParams(spp=16, sampler="sobol", rfilter="box"), RenderParams(spp=8, sampler="independent", rfilter="gaussian", max_depth=3)):
        fo, so = o.render(rp)
        fg, sg = g.render(rp, parity=True)
        assert rel_l2(api.develop(fg), O.develop(fo)) <= 3e-4
        assert abs(sg["rays"] - so["rays"]) <= 1e-3 * so["rays"] and abs(sg["path_length_sum"] - so["pathLengthSum"]) <= 1e-3 * so["pathLengthSum"]
    # throughput build (plane-form triangles, fast math): a ray that lands on the other side of an edge changes a whole path, whose
    # weight in the image falls with the sample count -- compared at 64 spp
    rp = RenderParams(spp=64, sampler="sobol", rfilter="box")
    fo, _ = o.render(rp)
    fg2, _ = g.render(rp, parity=False)
    assert rel_l2(api.develop(fg2), O.develop(fo)) <= REL_L2_TOL


def test_instancing_matches_flattened_geometry(b2ctx):
    """The same geometry once as instances, once flattened into world space: images agree to float rounding of the transforms."""
    from mitsuba_b200.scene import stress_scene
    a = stress_scene(6, 24, 24, 64, 64, instanced=True)
    b = stress_scene(6, 24, 24, 64, 64, instanced=False)
    for m in b.meshes:
        if m.name.startswith("inst"):
            m.bsdf = a.meshes[0].bsdf
    rp = RenderParams(spp=16, sampler="sobol", rfilter="box")
    fa, sa = api.Scene(b2ctx, a).render(rp, parity=True)
    fb, sb = api.Scene(b2ctx, b).render(rp, parity=True)
    assert rel_l2(api.develop(fa), api.develop(fb)) < 5e-3
    assert abs(sa["path_length_sum"] - sb["path_length_sum"]) <= 2e-3 * sb["path_length_sum"]
    assert sa["n_triangles"] * 5 < sb["n_triangles"]


def test_instancing_errors(b2ctx):
    from mitsuba_b200.scene import stress_scene
    d = stress_scene(2, 8, 8, 16, 16, instanced=True)
    d.meshes[0].radiance = (1.0, 1.0, 1.0)
    with pytest.raises(api.B2Error, match="Instancing of emitters"):
        api.Scene(b2ctx, d)
    d = stress_scene(2, 8, 8, 16, 16, instanced=True)
    g = api.Scene(b2ctx, d)
    with pytest.raises(api.B2Error, match="instanced geometry"):
        g.render(RenderParams(spp=1, integrator="volpath"))


def test_thinlens_sensor_parity(b2ctx):
    """<sensor type="thinlens"> (src/sensors/thinlens.cpp:327-350): aperture sample on Sobol' dimensions 2, 3; rays start on the lens."""
    d = cornell_box(64, 64)
    d.camera = dataclasses.replace(d.camera, aperture_radius=25.0, focus_distance=1100.0)
    g, o = pair(b2ctx, d)
    for smp in ("sobol", "independent"):
        rp = RenderParams(spp=16, sampler=smp, rfilter="box")
        fo, so = o.render(rp)
        fg, sg = g.render(rp, parity=True)
        assert rel_l2(api.develop(fg), O.develop(fo)) <= 3e-4
        assert abs(sg["rays"] - so["rays"]) <= 1e-3 * so["rays"]
    fg2, _ = g.render(RenderParams(spp=16, sampler="sobol", rfilter="box"), parity=False)
    fo, _ = o.render(RenderParams(spp=16, sampler="sobol", rfilter="box"))
    assert rel_l2(api.develop(fg2), O.develop(fo)) <= REL_L2_TOL
    # and it differs from the pinhole image
    gp = api.Scene(b2ctx, cornell_box(64, 64))
    fp, _ = gp.render(RenderParams(spp=16, sampler="sobol", rfilter="box"), parity=True)
    assert rel_l2(api.develop(fg), api.develop(fp)) > 0.02
