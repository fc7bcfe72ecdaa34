"""Rates of the `direct` integrator (k_direct) next to `path` on the same scenes, 1024x1024, throughput build, one GPU.  Prints the card
(name, power limit, maximum SM clock) and then one JSON object per render: Msamples/s and ray queries per second (closest-hit +
occlusion queries over the CUDA-event time of the render).  On Cornell, `direct` (1,1) renders the image of `path` to depth 2; the two
are alternated so that both see the same state of a shared card.

    python scripts/bench_direct.py [cornell c3 env tex inst]
"""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mitsuba_b200 import api
from mitsuba_b200.scene import RenderParams, config3_scene, cornell_box, envmap_scene, stress_scene, textured_scene


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True, timeout=30)
    name, power, smax, sm = [c.strip() for c in r.stdout.strip().split(",")]
    return {"card": name, "power_limit_w": float(power), "sm_max_mhz": float(smax), "sm_clock_mhz_idle": float(sm)}


def rate(label, sc, rp, reps=3):
    sc.render(RenderParams(**{**rp.__dict__, "spp": min(rp.spp, 4)}))   # warm-up: modules, first launch of every kernel the render uses
    best = None
    for _ in range(reps):
        _, st = sc.render(rp)
        if best is None or st["ms_total"] < best["ms_total"]:
            best = st
    ms = best["ms_total"]
    out = dict(run=label, integrator=rp.integrator, counts=[rp.emitter_samples, rp.bsdf_samples] if rp.integrator == "direct" else None,
               max_depth=rp.max_depth if rp.integrator == "path" else None, spp=rp.spp, rfilter=rp.rfilter, ms=round(ms, 2),
               msamples_s=round(best["samples"] / ms / 1e3, 1), mrays_s=round((best["rays"] + best["shadow_rays"]) / ms / 1e3, 1),
               rays_per_sample=round(best["rays"] / best["samples"], 3), shadow_rays_per_sample=round(best["shadow_rays"] / best["samples"], 3),
               launches=best["kernel_launches"])
    print(json.dumps(out), flush=True)
    return out


def main():
    which = sys.argv[1:] or ["cornell", "c3", "env", "tex", "inst"]
    print(json.dumps(card()), flush=True)
    ctx = api.Context(0)
    D = lambda ne, nb, **k: RenderParams(integrator="direct", emitter_samples=ne, bsdf_samples=nb, **k)
    if "cornell" in which:
        sc = api.Scene(ctx, cornell_box(1024, 1024))
        for _ in range(2):   # alternated: direct (1,1) and path to depth 2 render the same image
            rate("cornell", sc, D(1, 1, spp=64, sampler="sobol", rfilter="box"))
            rate("cornell", sc, RenderParams(spp=64, sampler="sobol", rfilter="box", max_depth=2))
        rate("cornell", sc, D(4, 4, spp=64, sampler="sobol", rfilter="box"))
        rate("cornell", sc, RenderParams(spp=64, sampler="sobol", rfilter="box"))
        sc.close()
    for key, label, mk, kw, spp in (("c3", "config3_balls", lambda: config3_scene(1024, 1024), dict(sampler="sobol", rfilter="box"), 32),
                                    ("env", "envmap_balls", lambda: envmap_scene(1024, 1024), dict(sampler="sobol", rfilter="gaussian"), 32),
                                    ("tex", "textured_ball", lambda: textured_scene(1024, 1024, filter_type="ewa", tex_res=1024, n_theta=200, n_phi=200),
                                     dict(sampler="sobol", rfilter="gaussian"), 32),
                                    ("inst", "instances_10M", lambda: stress_scene(100, width=1024, height=1024, instanced=True),
                                     dict(sampler="sobol", rfilter="box"), 16)):
        if key not in which:
            continue
        sc = api.Scene(ctx, mk())
        rate(label, sc, D(1, 1, spp=spp, **kw))
        rate(label, sc, D(4, 4, spp=spp, **kw))
        rate(label, sc, RenderParams(spp=spp, max_depth=2, **kw))
        sc.close()
    ctx.close()


if __name__ == "__main__":
    main()
