"""The device renderer against films rendered by the REFERENCE's own code for the plugins that joined the assembled reference renderer
last (tests/golden/path_ref_ext.npz: src/sensors/thinlens.cpp, src/emitters/constant.cpp, src/shapes/{shapegroup,instance}.cpp inside
oracle/_ref/libpathref.so -- see tests/gen_golden.py).  No oracle in between: this is the reference's output.

Written after the round's GPU minutes were spent (the pin moved the constant emitter to the front of the emitter list in the host code,
b2_scene_commit): the file sorts behind the other device tests on purpose, so that a surprise here cannot mask them under `-x`."""
import os

import numpy as np
import pytest

import ref_pins
from mitsuba_b200 import api

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))

# Throughput build on these tiny fixtures: at most this fraction of pixels may hold a flipped path (the rest must agree to 1e-3 per pixel);
# media flip more (every Woodcock step compares against a random number)
FAST_OFF_FRACTION = 0.004
FAST_TOL = {"vol": 5e-2, "env": 5e-2}


def rel_l2(a, b):
    return float(np.sqrt(((a.astype(np.float64) - b) ** 2).sum() / (b.astype(np.float64) ** 2).sum()))


def test_device_images_of_thinlens_constant_emitter_and_instances_match_the_reference_renderer(b2ctx):
    g = np.load(os.path.join(HERE, "golden", "path_ref_ext.npz"))
    n = 0
    for name, desc, rp in ref_pins.image_cases_ext():
        ref = g[name + "/film"]
        sc = api.Scene(b2ctx, desc)
        film, st = sc.render(rp, parity=True)
        film = np.asarray(film).reshape(ref.shape)
        assert np.allclose(film[..., 4], ref[..., 4], rtol=1e-5, atol=1e-6), name            # weights: identical sample positions
        assert np.allclose(film[..., 3], ref[..., 3], rtol=1e-4, atol=1e-4), name            # alpha
        # identical sample sets and splats; what is left is libm (device sin/cos/exp/log vs glibc), the last bit of the camera matrix and,
        # for instances, the inverse matrices (exactly affine here, float Gauss-Jordan in the reference: 3e-4 on these images with the
        # oracle, tests/test_oracle_reference_pins.py).  volpath: a Woodcock walk compares density / max against a random number, so
        # libm rounding flips an occasional collision (same tolerance as tests/test_gpu_reference_images.py)
        tol = 2e-3 if name == "env_volpath_smoke" else 3e-3 if name.startswith("instances") else 1e-3 if name.startswith("crop") else 3e-4   # crop: 43 x 33 pixels, one flipped path weighs 5e-4
        assert rel_l2(film[..., :3], ref[..., :3]) <= tol, (name, rel_l2(film[..., :3], ref[..., :3]))
        # the throughput build (FMA contraction, --use_fast_math, plane-form triangles; the build bench.py times) against the same
        # reference film: identical sample positions (weights), and every pixel within 1e-3 of the reference except the handful whose
        # path was flipped by an ulp-level difference (one flipped path moves a pixel of these 4-16 spp fixtures by percents; rough
        # dielectrics flip the most paths, diffuse scenes the fewest)
        fast = np.asarray(sc.render(rp, parity=False)[0]).reshape(ref.shape)
        assert np.allclose(fast[..., 4], ref[..., 4], rtol=1e-5, atol=1e-6), name
        rel = np.abs(fast[..., :3] - ref[..., :3]).max(-1) / np.maximum(np.abs(ref[..., :3]).max(-1), 1e-3 * ref[..., :3].max())
        n_off = int((rel > 1e-3).sum())
        if "vol" not in name:
            # (a gaussian splat spreads one flipped path over its 5 x 5 footprint)
            assert n_off <= max(4, int(FAST_OFF_FRACTION * rel.size)) * (12 if rp.rfilter == "gaussian" else 1), (name, n_off, rel.size)
        assert rel_l2(fast[..., :3], ref[..., :3]) <= FAST_TOL.get(name.split("_")[0], 2e-2), (name, rel_l2(fast[..., :3], ref[..., :3]))
        sc.close()
        n += 1
    assert n == 11


def test_device_emitter_selection_puts_the_constant_emitter_first(b2ctx):
    """Scene::m_emitters order (scene.cpp:510-516 vs :322-335): with samplingWeight 2 : 1 the environment owns [0, 2/3) of the selection
    sample although the scene description lists it after the area light.  Probe: b2_sample_emitter_direct against the reference's
    Scene::sampleEmitterDirect is covered on the CPU side; here the device probe must send small selection samples to the far sphere."""
    cases = {name: (desc, rp) for name, desc, rp in ref_pins.image_cases_ext()}
    desc, rp = cases["env_plus_area_cbox"]
    sc = api.Scene(b2ctx, desc)
    rng = np.random.default_rng(99)
    n = 400
    refp = np.zeros((n, 6), np.float32)
    refp[:, 0:3] = rng.uniform(50, 500, (n, 3))
    refp[:, 3:6] = ref_pins._dirs(rng, n)
    smp = rng.random((n, 2)).astype(np.float32)
    out = np.asarray(sc.sample_emitter_direct(refp, smp, parity=True)).reshape(n, 12)
    ok = out[:, 8] == 1
    far = np.linalg.norm(out[:, 9:12] - refp[:, 0:3], axis=1) > 700
    assert ok.sum() > 50
    assert far[ok & (smp[:, 0] < 0.6)].all() and not far[ok & (smp[:, 0] > 0.7)].any()
    sc.close()
