"""k_bounce_flat: a shared-memory resident scene shaded by one launch traces, shades and shadow-tests every path in one kernel per
iteration.  On a flat scene with two BSDF classes the default dispatch is class-sorted (k_extend_flat, one k_shade per class,
k_occluded_flat) while flags bit1 selects the bounce kernel with the generic shading instance: in the IEEE build both give the same
paths, so the per-pixel path statistics and the counters must match exactly and the films up to the order of the film atomics."""
import dataclasses

import numpy as np
import pytest

from mitsuba_b200 import api
from mitsuba_b200.scene import Bsdf, RenderParams, cornell_box

pytestmark = pytest.mark.gpu

COUNTERS = ("samples", "rays", "shadow_rays", "unoccluded_shadow_rays", "path_length_sum", "bad_samples", "dim_overflow")


def cornell_mixed(width, height, opened=False):
    """The Cornell box with the short block a GGX rough conductor (two BSDF classes, still one flat leaf).  `opened`: without the red
    wall, lit by a constant environment as well."""
    d = cornell_box(width, height)
    for m in d.meshes:
        if m.name == "short":
            m.bsdf = Bsdf("roughconductor", distribution="ggx", alpha_u=0.2, alpha_v=0.2, eta=(0.2004, 0.9240, 1.1022), k=(3.9129, 2.4528, 2.1421))
    if opened:
        d.meshes = [m for m in d.meshes if m.name != "left"]
        d.env_radiance = (0.4, 0.5, 0.6)
    return d


def rel_l2(a, b):
    return float(np.sqrt(((a - b) ** 2).sum() / max((b ** 2).sum(), 1e-30)))


CASES = {
    "sobol_box": dict(rp=RenderParams(spp=16, sampler="sobol", rfilter="box")),
    "sobol_gaussian": dict(rp=RenderParams(spp=16, sampler="sobol", rfilter="gaussian")),
    "independent": dict(rp=RenderParams(spp=16, sampler="independent", rfilter="gaussian")),
    "max_depth_2": dict(rp=RenderParams(spp=16, sampler="sobol", rfilter="box", max_depth=2)),
    "hide_emitters": dict(rp=RenderParams(spp=16, sampler="sobol", rfilter="box", hide_emitters=True)),
    "strict_normals": dict(rp=RenderParams(spp=16, sampler="sobol", rfilter="box", strict_normals=True)),
    "crop": dict(rp=RenderParams(spp=16, sampler="sobol", rfilter="gaussian"), crop=(40, 24, 72, 80)),
    "opened_constant_env": dict(rp=RenderParams(spp=16, sampler="sobol", rfilter="gaussian"), opened=True),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_bounce_matches_class_sorted_dispatch(b2ctx, case):
    c = CASES[case]
    d = cornell_mixed(128, 128, opened=c.get("opened", False))
    if "crop" in c:
        d.camera = dataclasses.replace(d.camera, crop=c["crop"])
    g = api.Scene(b2ctx, d)
    f_sorted, s_sorted = g.render(c["rp"], parity=True, flags=32 | 4)
    p_sorted = g.pixel_stats()
    f_bounce, s_bounce = g.render(c["rp"], parity=True, flags=32 | 4 | 2)
    p_bounce = g.pixel_stats()
    assert s_sorted["ms_extend"] > 0 and s_bounce["ms_extend"] == 0 and s_bounce["ms_occluded"] == 0   # the two dispatches really differ
    assert np.array_equal(p_sorted, p_bounce), (case, int((p_sorted != p_bounce).sum()))
    for k in COUNTERS:
        assert s_sorted[k] == s_bounce[k], (case, k, s_sorted[k], s_bounce[k])
    assert s_bounce["samples"] == f_bounce.shape[0] * f_bounce.shape[1] * 16
    assert rel_l2(np.asarray(f_bounce, np.float64), np.asarray(f_sorted, np.float64)) <= 1e-6, case
    g.close()


@pytest.fixture(scope="module")
def cbox(b2ctx):
    g = api.Scene(b2ctx, cornell_box(128, 128))
    yield g
    g.close()


@pytest.mark.parametrize("parity", [True, False])
def test_single_class_cornell_runs_one_kernel_per_bounce(cbox, parity):
    rp = RenderParams(spp=16, sampler="sobol", rfilter="box")
    _, st = cbox.render(rp, parity=parity, flags=4)
    assert st["kernel_launches"] == 3 * st["iterations"] + 1   # publish, generate, bounce (+ the film pack)
    assert st["ms_extend"] == 0 and st["n_extend"] == 0 and st["ms_occluded"] == 0 and st["n_occluded"] == 0
    assert st["ms_shade"] > 0 and st["n_shade"] == st["iterations"]
    assert 0 < st["unoccluded_shadow_rays"] <= st["shadow_rays"] < st["rays"]
    _, se = cbox.render(rp, parity=parity, flags=8)   # plain launches bracketed by CUDA events: the bounce kernel is timed as stage 2
    assert se["n_extend"] == 0 and se["n_occluded"] == 0 and se["n_shade"] == se["iterations"]
    for k in COUNTERS:
        assert st[k] == se[k], k


def test_throughput_build_changes_few_paths(cbox):
    rp = RenderParams(spp=16, sampler="sobol", rfilter="box")
    _, sp = cbox.render(rp, parity=True, flags=32)
    pp = cbox.pixel_stats()
    _, sf = cbox.render(rp, parity=False, flags=32)
    pf = cbox.pixel_stats()
    assert sp["samples"] == sf["samples"]
    assert (pp != pf).sum() <= 2e-4 * sp["samples"], int((pp != pf).sum())
