"""k_bounce_flat keeps each path of a shared-memory resident scene in registers until it ends (or until its per-launch vertex budget
runs out, when it is parked in the pool and continued by the next launch), and k_generate drains that route's pool in slot order.
So one iteration renders about one pool's worth of samples, and the same (pixel, sample) paths come out as through the class-sorted
kernels, which advance every path by one vertex per iteration."""
import numpy as np
import pytest

from mitsuba_b200 import api
from mitsuba_b200.scene import Bsdf, RenderParams, cornell_box

pytestmark = pytest.mark.gpu

COUNTERS = ("samples", "rays", "shadow_rays", "unoccluded_shadow_rays", "path_length_sum", "bad_samples", "dim_overflow")
POOL = 4096


def rel_l2(a, b):
    return float(np.sqrt(((a - b) ** 2).sum() / max((b ** 2).sum(), 1e-30)))


def bright_mixed_box(width, height):
    """The Cornell box with every diffuse wall at 0.95 reflectance, so that some thousands of its paths run past the per-launch vertex
    budget (16) and are parked and continued, and the short block a GGX rough conductor, so that the default dispatch is class-sorted
    and flags bit1 selects k_bounce_flat."""
    d = cornell_box(width, height)
    for m in d.meshes:
        if m.radiance is not None:
            continue
        if m.name == "short":
            m.bsdf = Bsdf("roughconductor", distribution="ggx", alpha_u=0.2, alpha_v=0.2, eta=(0.2004, 0.9240, 1.1022), k=(3.9129, 2.4528, 2.1421))
        else:
            m.bsdf = Bsdf("diffuse", reflectance=(0.95, 0.95, 0.95))
    return d


@pytest.fixture(scope="module")
def cbox(b2ctx):
    g = api.Scene(b2ctx, cornell_box(128, 128))
    yield g
    g.close()


@pytest.mark.parametrize("parity", [True, False])
def test_one_iteration_renders_about_one_pool_of_samples(cbox, parity):
    rp = RenderParams(spp=16, sampler="sobol", rfilter="box")
    _, st = cbox.render(rp, parity=parity, pool_size=POOL, flags=4)
    assert st["pool_size"] == POOL
    assert st["samples"] == 128 * 128 * 16
    full = st["samples"] // POOL
    # a few more for the paths parked by the vertex budget and the last, partly filled iterations, and up to B2_RING - 1 = 63 that the
    # host had queued ahead of the device when it saw the render end (they run on an empty pool); one vertex per path and iteration
    # would take about rays / samples (~4) times as many
    assert full <= st["iterations"] <= full + 8 + 63, (st["iterations"], full)
    assert st["kernel_launches"] == 3 * st["iterations"] + 1
    assert 0 < st["unoccluded_shadow_rays"] <= st["shadow_rays"] < st["rays"]


def test_parked_paths_match_class_sorted_dispatch(b2ctx):
    g = api.Scene(b2ctx, bright_mixed_box(96, 96))
    rp = RenderParams(spp=16, sampler="sobol", rfilter="box")
    f_sorted, s_sorted = g.render(rp, parity=True, pool_size=POOL, flags=32 | 4)
    p_sorted = g.pixel_stats()
    f_res, s_res = g.render(rp, parity=True, pool_size=POOL, flags=32 | 4 | 2)
    p_res = g.pixel_stats()
    assert s_sorted["ms_extend"] > 0 and s_res["ms_extend"] == 0 and s_res["ms_occluded"] == 0   # the two dispatches really differ
    # longer paths than in the Cornell box (3.55 vertices on average)
    assert s_res["path_length_sum"] / s_res["samples"] > 4.5
    assert s_res["iterations"] < s_sorted["iterations"]
    assert np.array_equal(p_sorted, p_res), int((p_sorted != p_res).sum())
    for k in COUNTERS:
        assert s_sorted[k] == s_res[k], (k, s_sorted[k], s_res[k])
    assert s_res["samples"] == 96 * 96 * 16
    assert rel_l2(np.asarray(f_res, np.float64), np.asarray(f_sorted, np.float64)) <= 1e-6
    g.close()


def test_resident_route_is_deterministic_in_its_paths(cbox):
    """Which slot renders which (pixel, sample) depends on atomics; the paths themselves do not."""
    rp = RenderParams(spp=16, sampler="independent", rfilter="gaussian")
    _, s1 = cbox.render(rp, parity=True, pool_size=POOL, flags=32)
    p1 = cbox.pixel_stats()
    _, s2 = cbox.render(rp, parity=True, flags=32)
    p2 = cbox.pixel_stats()
    assert np.array_equal(p1, p2)
    for k in COUNTERS:
        assert s1[k] == s2[k], k
