"""The device renderer against images rendered by the REFERENCE's own code (tests/golden/path_ref.npz: MIPathTracer::Li, renderBlock,
Scene, ShapeKDTree, sensor, emitter, Sobol' sampler, filters, ImageBlock and the BSDF plugins compiled from /root/reference into
oracle/_ref/libpathref.so -- see tests/gen_golden.py).  No oracle in between: this is the reference's output."""
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
FAST_TOL = {"vol": 5e-2}


def rel_l2(a, b):
    return float(np.sqrt(((a.astype(np.float64) - b) ** 2).sum() / (b.astype(np.float64) ** 2).sum()))


def test_device_images_match_the_reference_renderer(b2ctx):
    g = np.load(os.path.join(HERE, "golden", "path_ref.npz"))
    n = 0
    for name, desc, rp in ref_pins.image_cases():
        ref = g[name + "/film"]
        sc = api.Scene(b2ctx, desc)
        film, st = sc.render(rp, parity=True)
        film = np.asarray(film).reshape(ref.shape)
        # identical sample sets and splats; what is left is libm (device sin/cos/exp vs glibc) and the last bit of the camera matrix
        assert np.allclose(film[..., 4], ref[..., 4], rtol=1e-5, atol=1e-6), name            # weights
        assert np.allclose(film[..., 3], ref[..., 3], rtol=1e-4, atol=1e-4), name            # alpha
        # volpath: a Woodcock walk compares density / max against a random number, so device libm rounding flips an occasional collision
        tol = 2e-3 if name.startswith("vol_h") else 3e-4
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
    assert n == 19
