"""The oracle of the `direct` integrator (tests/orc_direct.cpp) against the reference's own src/integrators/direct/direct.cpp.

tests/golden/path_ref_direct.npz holds films rendered by the renderer assembled from the reference's sources (oracle/path_ref_shim.cpp +
tests/direct_ref_shim.cpp: MIDirectIntegrator with the reference's Sobol' sampler, or this repository's counter stream served through the
Sampler interface, whose 2-D sample arrays follow the definition in DESIGN.md section 8f; written by `python tests/direct_pins.py`).  The
oracle must reproduce every film bit for bit."""
import dataclasses
import os

import numpy as np
import pytest

from direct_pins import DirectOracle, image_cases_direct
from mitsuba_b200.scene import Bsdf, RenderParams, cornell_box, material_ball

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "path_ref_direct.npz")


def oracle_scene(desc, g, name):
    """The oracle scene of fixture case `name`, with the camera / instance / environment-map matrices the reference derived."""
    if (name + "/env_to_local") in g.files:
        desc.envmap = dataclasses.replace(desc.envmap, to_local=g[name + "/env_to_local"])
    inv = g[name + "/instance_inverses"] if (name + "/instance_inverses") in g.files else None
    return DirectOracle(desc, sample_to_camera=g[name + "/s2c"], instance_inverses=inv)


def test_oracle_direct_films_match_the_reference_renderer_golden():
    g = np.load(GOLDEN)
    names = []
    for name, desc, rp in image_cases_direct():
        ref = g[name + "/film"]
        film = np.asarray(oracle_scene(desc, g, name).render(rp)[0]).reshape(ref.shape)
        assert np.array_equal(film, ref), (name, float(np.abs(film - ref).max()))
        assert ref[..., :3].max() > 0.01 and ref[..., 4].min() > 0, name
        names.append(name)
    assert len(names) == 22
    # the cases cover what the arrays change: counts (1,1), (4,2), (3,0), (0,2) on both samplers and a thin lens
    assert {"direct_cbox_11_sobol_box", "direct_cbox_42_sobol_gaussian", "direct_cbox_30_counter_box", "direct_cbox_02_counter_gaussian",
            "direct_thinlens_42_sobol", "direct_thinlens_13_sobol", "direct_thinlens_51_counter"} <= set(names)


def _open_box_with_sky(w, h):
    d = cornell_box(w, h)
    d.meshes = [m for i, m in enumerate(d.meshes) if i != 1]   # open the box: the constant emitter is seen and sampled
    d.env_radiance = (0.4, 0.6, 1.0)
    d.env_sampling_weight = 2.0
    return d


@pytest.mark.parametrize("sampler", ["sobol", "independent"])
@pytest.mark.parametrize("scene", ["cbox", "cbox_sky"])
def test_direct_11_is_path_to_depth_2_sample_for_sample(scene, sampler):
    """On scenes where every BSDF has a smooth lobe, `direct` with one sample of each strategy and `path` with maxDepth = 2 draw the same
    numbers (camera 0-1, emitter sample 2-3, BSDF sample 5-6), weigh by MIS weights that differ only by the exact factors 1/2 (both
    densities) and 1 (the count weight), and add the emitter and environment terms in the same order: every sample is bit-identical."""
    desc = cornell_box(32, 32) if scene == "cbox" else _open_box_with_sky(32, 32)
    o = DirectOracle(desc)
    fp, sp, pp = o.render(RenderParams(spp=4, sampler=sampler, rfilter="gaussian", max_depth=2), per_sample=True)
    fd, sd, pd = o.render(RenderParams(spp=4, sampler=sampler, rfilter="gaussian", integrator="direct"), per_sample=True)
    assert np.array_equal(pp, pd) and np.array_equal(fp, fd)
    assert sp["rays"] == sd["rays"] and sp["shadowRays"] == sd["shadowRays"] and sp["samples"] == sd["samples"]
    assert sd["pathLengthSum"] == 0 and pd[..., :3].max() > 0.1


def test_direct_draws_the_emitter_sample_on_delta_only_bsdfs():
    """`direct` draws its emitter sample before the ESmooth test (direct.cpp:210-214), `path` only behind it (path.cpp:173-176).  On a
    smooth conductor ball (delta-only, its sample is not read) the two still agree sample for sample; on a dielectric ball -- delta-only and
    sample-dependent -- the samples whose camera ray hits the ball take their BSDF sample from other dimensions: the images differ,
    and agree in the mean."""
    for bsdf, same in ((Bsdf("conductor"), True), (Bsdf("dielectric", int_ior=1.5), False)):
        o = DirectOracle(material_ball(bsdf, 16, 16, n_theta=12, n_phi=24))
        _, _, pp = o.render(RenderParams(spp=64, sampler="sobol", rfilter="box", max_depth=2), per_sample=True)
        _, _, pd = o.render(RenderParams(spp=64, sampler="sobol", rfilter="box", integrator="direct"), per_sample=True)
        eq = np.all(pp == pd, axis=-1)
        if same:
            assert eq.all()
        else:
            assert 0.2 < eq.mean() < 1.0
            a, b = pp[..., :3].mean(), pd[..., :3].mean()
            assert abs(a - b) < 0.1 * a


def test_direct_sample_arrays_are_counted_and_change_the_estimate():
    """Counts above 1 take their samples from the arrays: one closest-hit ray per BSDF sample, one shadow-ray candidate per emitter
    sample; a count of 0 still consumes its regular 2-D sample."""
    o = DirectOracle(cornell_box(16, 16))
    base = dict(integrator="direct", spp=4, sampler="sobol", rfilter="box")
    _, s11 = o.render(RenderParams(**base))
    _, s42 = o.render(RenderParams(**base, emitter_samples=4, bsdf_samples=2))
    _, s30 = o.render(RenderParams(**base, emitter_samples=3, bsdf_samples=0))
    n = s11["samples"]
    assert s30["rays"] == n                              # camera rays only
    assert s42["rays"] > s11["rays"] and s42["shadowRays"] > 3 * s11["shadowRays"]
