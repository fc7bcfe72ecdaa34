"""The set-up and tear-down that every integrator's render shares (b2_render): films written straight into device memory, cancelling
`direct`, and the stats an integrator reports after another integrator rendered the same scene."""
import ctypes as C
import threading
import time

import numpy as np
import pytest
import torch

from mitsuba_b200 import api
from mitsuba_b200.scene import RenderParams, cornell_box, smoke_scene, textured_scene

pytestmark = pytest.mark.gpu

COUNTERS = ("samples", "rays", "shadow_rays", "unoccluded_shadow_rays", "path_length_sum", "bad_samples", "dim_overflow")
STAGE_TIMES = ("ms_generate", "ms_extend", "ms_shade", "ms_occluded", "n_generate", "n_extend", "n_shade", "n_occluded")


def rel_l2(a, b):
    return float(np.sqrt(((a.astype(np.float64) - b) ** 2).sum() / (b.astype(np.float64) ** 2).sum()))


# box filter: every sample adds the same filter weight, so the weight channel does not depend on the order of the film atomics
DEVICE_FILM_CASES = {
    "path_cornell": (lambda: cornell_box(128, 128), RenderParams(spp=16, sampler="sobol", rfilter="box")),
    "volpath_smoke": (lambda: smoke_scene(64, 64, res=16), RenderParams(spp=8, sampler="sobol", rfilter="box", integrator="volpath")),
    "direct_cornell": (lambda: cornell_box(128, 128),
                       RenderParams(spp=16, sampler="sobol", rfilter="box", integrator="direct", emitter_samples=2, bsdf_samples=2)),
    "direct_textured": (lambda: textured_scene(64, 64, tex_res=64), RenderParams(spp=8, sampler="sobol", rfilter="box", integrator="direct")),
}


@pytest.mark.parametrize("case", sorted(DEVICE_FILM_CASES))
def test_device_film_matches_host_film(b2ctx, case):
    """film_on_device: the packed film lands in a CUDA tensor; it is the host film up to the order of the film atomics."""
    make, rp = DEVICE_FILM_CASES[case]
    sc = api.Scene(b2ctx, make())
    host, sh = sc.render(rp)
    film = torch.zeros((sc.H, sc.W, 5), dtype=torch.float32, device="cuda")
    _, sd = sc.render(rp, film=film)
    dev = film.cpu().numpy()
    for k in COUNTERS:
        assert sd[k] == sh[k], (k, sd[k], sh[k])
    assert np.allclose(dev[..., 4], host[..., 4], rtol=1e-6)
    assert rel_l2(dev[..., :3], host[..., :3]) <= 1e-6
    sc.close()


def test_cancel_direct_returns_status(b2ctx):
    """b2_cancel from another thread stops `direct` between two slices with B2_ERR_CANCELLED, and the scene keeps rendering."""
    d = cornell_box(512, 512)
    g = api.Scene(b2ctx, d)
    rp = RenderParams(spp=8192, sampler="sobol", rfilter="box", integrator="direct", emitter_samples=8, bsdf_samples=8)
    p = api.make_params(rp, False, 0, False, 0)
    film = np.zeros((512, 512, 5), np.float32)
    rc = {}
    t = threading.Thread(target=lambda: rc.setdefault("rc", g.L.b2_render(g.h, C.byref(p), film.ctypes.data_as(C.POINTER(C.c_float)))))
    t.start(); time.sleep(0.05)
    t0 = time.time()
    while t.is_alive() and time.time() - t0 < 60:   # b2_render clears the flag when it starts: keep asking until it lands
        g.L.b2_cancel(g.h); time.sleep(0.005)
    t.join(timeout=60)
    assert not t.is_alive() and rc["rc"] == 5
    f, s = g.render(RenderParams(spp=2, sampler="sobol", rfilter="box", integrator="direct"))
    assert s["samples"] == 512 * 512 * 2


def test_stats_do_not_leak_between_integrators(b2ctx):
    """Every render reports its own pool size, path lengths and stage times, whatever the scene rendered before."""
    sc = api.Scene(b2ctx, cornell_box(128, 128))
    rp = RenderParams(spp=16, sampler="sobol", rfilter="box")
    _, sp = sc.render(rp, flags=4)
    assert sp["pool_size"] > 0 and sp["path_length_sum"] > 0 and sp["n_shade"] > 0
    _, sd = sc.render(RenderParams(spp=16, sampler="sobol", rfilter="box", integrator="direct"), flags=4 | 8)
    for k in STAGE_TIMES:
        assert sd[k] == 0, (k, sd[k])
    assert sd["pool_size"] == 0 and sd["path_length_sum"] == 0
    assert sd["iterations"] >= 1 and sd["kernel_launches"] == sd["iterations"] + 1
    # plain launches timed by events (flags bit3): the resident route times one shading stage per iteration
    _, sp = sc.render(rp, flags=4 | 8)
    assert sp["pool_size"] > 0 and sp["n_shade"] == sp["iterations"]
    sc.close()
