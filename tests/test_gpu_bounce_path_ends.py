"""On the route of a shared-memory resident scene, k_generate writes only a fresh path's ray, sampler index, pixel and state word:
k_bounce_flat starts its throughput, eta and Li itself when it sees PF_FRESH, and a parked path (one that used up its per-launch vertex
budget) reloads them from the pool.  On a flat scene with two BSDF classes the default dispatch is class-sorted (k_extend_flat, one k_shade
per class, k_occluded_flat; k_generate writes all of a fresh path's records) while flags bit1 selects the bounce kernel.  In the IEEE
build both give the same paths, so the per-pixel path statistics and the counters must match exactly, and the films up to the order of
the film atomics, for paths that end at every depth limit and roulette setting, with and without a shadow ray at their last vertex."""
import numpy as np
import pytest

from mitsuba_b200 import api
from mitsuba_b200.scene import Bsdf, RenderParams, cornell_box

pytestmark = pytest.mark.gpu

COUNTERS = ("samples", "rays", "shadow_rays", "unoccluded_shadow_rays", "path_length_sum", "bad_samples", "dim_overflow")
W = H = 96
SPP = 16


def mixed_box(opened=False, bright=False):
    """The Cornell box with the short block a GGX rough conductor (two BSDF classes, still one flat leaf).  `opened`: without the red
    wall, lit by a constant environment as well, so that shadow rays toward the environment leave through the opening and the far side
    of the scene-box clip ends them.  `bright`: every diffuse wall at 0.95 reflectance, so that paths run past the vertex budget (16)."""
    d = cornell_box(W, H)
    for m in d.meshes:
        if m.name == "short":
            m.bsdf = Bsdf("roughconductor", distribution="ggx", alpha_u=0.2, alpha_v=0.2, eta=(0.2004, 0.9240, 1.1022), k=(3.9129, 2.4528, 2.1421))
        elif bright and m.radiance is None:
            m.bsdf = Bsdf("diffuse", reflectance=(0.95, 0.95, 0.95))
    if opened:
        d.meshes = [m for m in d.meshes if m.name != "left"]
        d.env_radiance = (0.4, 0.5, 0.6)
    return d


def rel_l2(a, b):
    return float(np.sqrt(((a - b) ** 2).sum() / max((b ** 2).sum(), 1e-30)))


# maxDepth 1 ends every path at its first vertex (no shadow ray), 2 and 3 end paths right after a vertex that emitted one; rrDepth 1 lets
# Russian roulette end paths from the second vertex on
CASES = {f"max_depth_{md}_rr_{rr}": dict(rp=RenderParams(spp=SPP, sampler="sobol", rfilter="box", max_depth=md, rr_depth=rr))
         for md in (1, 2, 3, -1) for rr in (1, 5)}
CASES.update({
    "hide_emitters": dict(rp=RenderParams(spp=SPP, sampler="sobol", rfilter="box", hide_emitters=True)),
    "strict_normals": dict(rp=RenderParams(spp=SPP, sampler="sobol", rfilter="box", strict_normals=True)),
    "opened_constant_env": dict(rp=RenderParams(spp=SPP, sampler="sobol", rfilter="gaussian"), opened=True),
    # a 4096-slot pool: many launches, and parked paths continue in later ones
    "bright_parked": dict(rp=RenderParams(spp=SPP, sampler="sobol", rfilter="box"), bright=True, pool=4096),
})


@pytest.mark.parametrize("case", sorted(CASES))
def test_bounce_path_ends_match_class_sorted_dispatch(b2ctx, case):
    c = CASES[case]
    g = api.Scene(b2ctx, mixed_box(opened=c.get("opened", False), bright=c.get("bright", False)))
    pool = c.get("pool", 0)
    f_sorted, s_sorted = g.render(c["rp"], parity=True, pool_size=pool, flags=32 | 4)
    p_sorted = g.pixel_stats()
    f_bounce, s_bounce = g.render(c["rp"], parity=True, pool_size=pool, flags=32 | 4 | 2)
    p_bounce = g.pixel_stats()
    assert s_sorted["ms_extend"] > 0 and s_bounce["ms_extend"] == 0 and s_bounce["ms_occluded"] == 0   # the two dispatches really differ
    assert np.array_equal(p_sorted, p_bounce), (case, int((p_sorted != p_bounce).sum()))
    for k in COUNTERS:
        assert s_sorted[k] == s_bounce[k], (case, k, s_sorted[k], s_bounce[k])
    assert s_bounce["samples"] == W * H * SPP
    if c["rp"].max_depth != 1:
        assert 0 < s_bounce["unoccluded_shadow_rays"] < s_bounce["shadow_rays"]
    if c.get("bright"):
        assert s_bounce["path_length_sum"] / s_bounce["samples"] > 4.5   # longer paths than the budget allows some of them
    assert rel_l2(np.asarray(f_bounce, np.float64), np.asarray(f_sorted, np.float64)) <= 1e-6, case
    g.close()


def test_throughput_build_bounce_changes_few_paths(b2ctx):
    """In the throughput build FMA contraction and the fast intrinsics may round the shading code of the two dispatches differently, so
    a few paths may part; the films stay within the build's image tolerance."""
    g = api.Scene(b2ctx, mixed_box())
    rp = RenderParams(spp=SPP, sampler="sobol", rfilter="box")
    f_sorted, s_sorted = g.render(rp, parity=False, flags=32 | 4)
    p_sorted = g.pixel_stats()
    f_bounce, s_bounce = g.render(rp, parity=False, flags=32 | 4 | 2)
    p_bounce = g.pixel_stats()
    assert s_sorted["samples"] == s_bounce["samples"] == W * H * SPP
    assert (p_sorted != p_bounce).sum() <= 2e-4 * s_bounce["samples"], int((p_sorted != p_bounce).sum())
    assert rel_l2(np.asarray(f_bounce, np.float64), np.asarray(f_sorted, np.float64)) <= 1e-3
    g.close()
