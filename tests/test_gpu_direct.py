"""The `direct` integrator on the device (k_direct) against films rendered by the reference's own MIDirectIntegrator
(tests/golden/path_ref_direct.npz, see tests/gen_golden.py) and against the oracle's counters; `direct` with one sample of each strategy
against the device's `path` to depth 2; shards; the scene-file route; the parameter checks of b2_render."""
import os
import re
import shutil

import numpy as np
import pytest

from direct_pins import DirectOracle, image_cases_direct
from mitsuba_b200 import api
from mitsuba_b200.scene import RenderParams, cornell_box, textured_scene
from oracle import oracle_api as O

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def rel_l2(a, b):
    return float(np.sqrt(((a.astype(np.float64) - b) ** 2).sum() / (b.astype(np.float64) ** 2).sum()))


def tolerance(name, parity):
    """Relative L2 of a device film against the reference's film of fixture case `name`."""
    # instances: the reference's float Gauss-Jordan inverses vs this repository's exactly affine ones (test_gpu_z_reference_images_ext.py)
    if name.startswith("direct_instances"):
        return 3e-3
    # texture / environment-map films: device libm in the filtered look-ups (as tests/test_gpu_texture.py and test_gpu_envmap.py allow)
    if name.startswith(("direct_tex", "direct_envmap")):
        # throughput build: every shading point of `direct` is an EWA look-up, whose fast-math weights differ by more than 1e-3 on a few
        # percent of look-ups (test_gpu_texture.py); on this 36 x 36 @ 4 spp film they do not average out.  The 1e-3 budget of the
        # throughput build is held on a larger render in test_device_direct_throughput_build_on_textures
        return 1e-3 if parity else 5e-3
    return 3e-4 if parity else 1e-3


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(HERE, "golden", "path_ref_direct.npz"))


def test_device_direct_matches_the_reference_renderer(b2ctx, golden):
    n, bad = 0, []
    for name, desc, rp in image_cases_direct():
        ref = golden[name + "/film"]
        sc = api.Scene(b2ctx, desc)
        fo, so = DirectOracle(desc, sample_to_camera=sc.sample_to_camera()).render(rp)
        for parity in (True, False):
            film, st = sc.render(rp, parity=parity)
            film = np.asarray(film).reshape(ref.shape)
            err = rel_l2(film[..., :3], ref[..., :3])
            # ray counters against the oracle (the IEEE restatement): the parity build to 1e-4; in the throughput build an ulp-level
            # difference of a hit point can flip an emitter sample to the back side of the light (no shadow ray) on a few samples
            ctol = 1e-4 if parity else 1e-3
            checks = {"weights": np.allclose(film[..., 4], ref[..., 4], rtol=1e-5, atol=1e-6),   # identical sample positions
                      "rgb": err <= tolerance(name, parity),
                      "samples": st["samples"] == so["samples"],
                      "rays": abs(st["rays"] - so["rays"]) <= ctol * so["rays"],
                      "shadow_rays": abs(st["shadow_rays"] - so["shadowRays"]) <= ctol * max(1, so["shadowRays"]),
                      "stats": st["path_length_sum"] == 0 and st["bad_samples"] == 0 and st["pool_size"] == 0}
            bad += [(name, parity, k, err, (st["rays"], so["rays"]), (st["shadow_rays"], so["shadowRays"])) for k, ok in checks.items() if not ok]
        sc.close()
        n += 1
    assert not bad, bad
    assert n == 22


def test_device_direct_throughput_build_on_textures(b2ctx):
    """The throughput build's budget (1e-3 relative L2, as tests/test_gpu_texture.py holds `path` to) on a textured render large enough for
    the fast-math EWA weights to average out, against the oracle."""
    d = textured_scene(96, 96, filter_type="ewa", tex_res=128)
    sc = api.Scene(b2ctx, d)
    rp = RenderParams(spp=64, sampler="sobol", rfilter="box", integrator="direct", emitter_samples=2, bsdf_samples=2)
    fo, _ = DirectOracle(d, sample_to_camera=sc.sample_to_camera()).render(rp)
    ff, _ = sc.render(rp, parity=False)
    assert rel_l2(api.develop(ff), O.develop(fo)) <= 1e-3
    sc.close()


def test_device_direct_11_is_device_path_to_depth_2(b2ctx):
    """One emitter and one BSDF sample per camera hit draw the numbers `path` draws to depth 2 and weigh them by the same MIS weights up to
    exact factors (tests/test_oracle_direct.py): the dedicated kernel must give path's counters and, up to the order of the film
    atomics, its film."""
    sc = api.Scene(b2ctx, cornell_box(128, 128))
    for sampler in ("sobol", "independent"):
        fp, sp = sc.render(RenderParams(spp=16, sampler=sampler, rfilter="gaussian", max_depth=2), parity=True)
        fd, sd = sc.render(RenderParams(spp=16, sampler=sampler, rfilter="gaussian", integrator="direct"), parity=True)
        for k in ("samples", "rays", "shadow_rays", "unoccluded_shadow_rays"):
            assert sp[k] == sd[k], (sampler, k, sp[k], sd[k])
        assert rel_l2(api.develop(fd), api.develop(fp)) <= 1e-6
        ff, _ = sc.render(RenderParams(spp=16, sampler=sampler, rfilter="gaussian", integrator="direct"), parity=False)
        assert rel_l2(api.develop(ff), api.develop(fp)) <= 1e-3
    sc.close()


@pytest.mark.parametrize("sampler", ["sobol", "independent"])
def test_device_direct_shards_add_up(b2ctx, sampler):
    """An array entry depends only on (pixel, sample, entry): samples [0, s/2) + [s/2, s) are the render of [0, s)."""
    sc = api.Scene(b2ctx, cornell_box(64, 48))
    rp = RenderParams(spp=8, sampler=sampler, rfilter="gaussian", integrator="direct", emitter_samples=4, bsdf_samples=2)
    full, sf = sc.render(rp, parity=True)
    a, sa = sc.render(RenderParams(**{**rp.__dict__, "sample_lo": 0, "sample_hi": 4}), parity=True)
    b, sb = sc.render(RenderParams(**{**rp.__dict__, "sample_lo": 4, "sample_hi": 8}), parity=True)
    assert sa["samples"] + sb["samples"] == sf["samples"] and sa["rays"] + sb["rays"] == sf["rays"]
    assert np.allclose(a[..., 4] + b[..., 4], full[..., 4], rtol=1e-6)
    assert rel_l2(a[..., :3] + b[..., :3], full[..., :3]) <= 1e-6
    sc.close()


def _cbox_xml(tmp_path, integrator):
    src = open(os.path.join(ROOT, "scenes", "cbox.xml")).read()
    text = re.sub(r'<integrator type="path">.*?</integrator>', integrator, src, flags=re.S)
    shutil.copytree(os.path.join(ROOT, "scenes", "meshes"), tmp_path / "meshes", dirs_exist_ok=True)
    p = tmp_path / "direct.xml"
    p.write_text(text)
    return str(p)


def test_xml_direct_route(b2ctx, tmp_path):
    path = _cbox_xml(tmp_path, '<integrator type="direct"><integer name="shadingSamples" value="4"/><integer name="bsdfSamples" value="2"/>'
                               '<boolean name="hideEmitters" value="true"/></integrator>')
    sc, rp = b2ctx.load_xml(path, ["spp=8", "res=48"])
    assert rp.integrator == "direct" and rp.emitter_samples == 4 and rp.bsdf_samples == 2 and rp.hide_emitters
    film, st = sc.render(rp, parity=True)
    fo, so = DirectOracle(cornell_box(48, 48), sample_to_camera=sc.sample_to_camera()).render(rp)
    assert st["samples"] == so["samples"] and abs(st["rays"] - so["rays"]) <= 1e-4 * so["rays"]
    assert rel_l2(api.develop(film), O.develop(fo)) < 3e-4
    sc.close()


def test_direct_parameter_errors(b2ctx, tmp_path):
    sc = api.Scene(b2ctx, cornell_box(16, 16))
    base = dict(spp=4, sampler="sobol", rfilter="box", integrator="direct")
    for kw, msg in ((dict(emitter_samples=-1), "must not be negative"), (dict(bsdf_samples=-2), "must not be negative"),
                    (dict(emitter_samples=0, bsdf_samples=0), "must be positive"),
                    (dict(spp=1 << 18, emitter_samples=1 << 14), "below 2\\^32")):
        with pytest.raises(api.B2Error, match=msg):
            sc.render(RenderParams(**{**base, **kw}))
    for flags in (32, 64):
        with pytest.raises(api.B2Error, match="diagnostics"):
            sc.render(RenderParams(**base), flags=flags)
    with pytest.raises(api.B2Error, match="out of range"):
        sc.render(RenderParams(**base, emitter_samples=40000))
    sc.close()
    for bad, msg in (('<integrator type="direct"><integer name="maxDepth" value="3"/></integrator>', "unreferenced property"),
                     ('<integrator type="direct"><integer name="emitterSamples" value="-1"/></integrator>', "sample counts"),
                     ('<integrator type="bdpt"/>', "unsupported integrator")):
        with pytest.raises(api.B2Error, match=msg):
            b2ctx.load_xml(_cbox_xml(tmp_path, bad), ["spp=4", "res=16"])
