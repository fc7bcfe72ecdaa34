"""Secondary measurements (not the headline): other BASELINE configs at reduced size + isolated traversal numbers.
Prints one JSON object per line."""
import json, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from mitsuba_b200 import api
from mitsuba_b200.scene import Bsdf, RenderParams, cornell_box, material_ball, stress_scene, smoke_scene

ctx = api.Context(0)
HBM = json.load(open(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")))["hbm_gbs"] if os.path.exists(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")) else 6650.0
CU = dict(eta=(0.2004, 0.9240, 1.1022), k=(3.9129, 2.4528, 2.1421))


def render_rate(name, desc, rp, flags=4, reps=2, **kw):
    t = time.time(); sc = api.Scene(ctx, desc); tb = time.time() - t
    sc.render(rp, flags=flags, **kw)
    best = None
    for _ in range(reps):
        _, st = sc.render(rp, flags=flags, **kw)
        if best is None or st["ms_total"] < best["ms_total"]:
            best = st
    n = desc.camera.width * desc.camera.height * rp.spp
    out = dict(scene=name, tris=desc.n_triangles(), bvh_nodes=best["n_bvh_nodes"], commit_s=round(tb, 3), res=desc.camera.width, spp=rp.spp, rfilter=rp.rfilter,
               msamples_s=round(n / best["ms_total"] / 1e3, 1), ms=round(best["ms_total"], 2), L=round(best["path_length_sum"] / best["samples"], 3),
               rays_per_sample=round(best["rays"] / best["samples"], 3),
               kernel_ms={k: round(best["ms_" + k], 2) for k in ("generate", "extend", "shade", "occluded")}, iters=best["iterations"], **kw)
    print(json.dumps(out), flush=True)
    return sc


def chord_rays(n, center, radius, seed=0):
    """kdbench-style incoherent rays: chords between uniform points on the bounding sphere (src/utils/kdbench.cpp:222-229)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    def sph():
        v = torch.randn((n, 3), device="cuda", generator=g); return v / v.norm(dim=1, keepdim=True)
    c = torch.tensor(center, device="cuda", dtype=torch.float32)
    a, b = c + radius * sph(), c + radius * sph()
    d = b - a; L = d.norm(dim=1, keepdim=True); d = d / L
    rays = torch.cat([a, torch.zeros((n, 1), device="cuda"), d, L], 1).contiguous().float()
    return rays


def trace_bench(name, sc, desc, n=1 << 22):
    P = np.concatenate([m.P for m in desc.meshes]); lo, hi = P.min(0), P.max(0)
    rays = chord_rays(n, (lo + hi) / 2, float(np.linalg.norm(hi - lo) / 2))
    out = torch.zeros((n, 4), device="cuda")
    for mode, label in ((0, "closest"), (1, "occlusion")):
        sc.trace_device(rays, out, n, mode=mode | 2)
        st = sc.stats()
        nv, pt = st["node_visits"] / n, st["prim_tests"] / n
        ms = min(sc.trace_device(rays, out, n, mode=mode) for _ in range(3))
        hits = float((out[:, 3].view(torch.int32) != (-1 if mode == 0 else 0)).float().mean()) if mode == 0 else float((out[:, 3].view(torch.int32) == 1).float().mean())
        ray_b = 48 if mode == 0 else 36
        alg = (ray_b + 64 * nv + 48 * pt) * n
        print(json.dumps(dict(trace=name, mode=label, rays=n, mrays_s=round(n / ms / 1e3, 1), ms=round(ms, 3), node_visits_per_ray=round(nv, 2),
                              tri_tests_per_ray=round(pt, 2), hit_frac=round(hits, 3), algorithmic_gbs=round(alg / ms / 1e6, 1), frac_of_hbm=round(alg / ms / 1e6 / HBM, 4))), flush=True)


which = sys.argv[1:] or ["cornell", "ball", "stress"]
if "cornell" in which:
    d = cornell_box(1024, 1024)
    sc = render_rate("cornell_box", d, RenderParams(spp=64, rfilter="gaussian"))
    render_rate("cornell_box", d, RenderParams(spp=64, rfilter="box"))
    render_rate("cornell_box", d, RenderParams(spp=64, rfilter="box", sampler="independent"))
    trace_bench("cornell_box", sc, d)
if "cornell_mixed" in which:
    # two BSDF classes in one flat leaf (the short block a GGX rough conductor): the class-sorted dispatch (k_extend_flat, one k_shade per
    # class, k_occluded_flat) against k_bounce_flat with the generic shading instance (flags bit1)
    d = cornell_box(1024, 1024)
    for m in d.meshes:
        if m.name == "short":
            m.bsdf = Bsdf("roughconductor", distribution="ggx", alpha_u=0.2, alpha_v=0.2, **CU)
    sc = render_rate("cornell_mixed/sorted", d, RenderParams(spp=64, rfilter="box"))
    render_rate("cornell_mixed/bounce", d, RenderParams(spp=64, rfilter="box"), flags=4 | 2)
if "ball" in which:
    for nm, b in (("roughconductor_ggx", Bsdf("roughconductor", distribution="ggx", alpha_u=0.1, alpha_v=0.1, **CU)),
                  ("roughdielectric_ggx", Bsdf("roughdielectric", distribution="ggx", alpha_u=0.1, alpha_v=0.1, int_ior="bk7", ext_ior="air")),
                  ("coating_roughconductor", Bsdf("coating", int_ior=1.5, ext_ior=1.0, nested=Bsdf("roughconductor", distribution="ggx", alpha_u=0.2, alpha_v=0.2, **CU)))):
        d = material_ball(b, 1024, 1024)
        sc = render_rate("material_ball/" + nm, d, RenderParams(spp=32, rfilter="gaussian"))
        if nm == "roughconductor_ggx":
            render_rate("material_ball/" + nm + "/unsorted", d, RenderParams(spp=32, rfilter="gaussian"), flags=4 | 2)
            trace_bench("material_ball", sc, d)
if "stress" in which:
    ninst = int(os.environ.get("STRESS_INSTANCES", "10"))
    d = stress_scene(ninst, width=1024, height=1024)
    sc = render_rate(f"stress_{ninst}x100k", d, RenderParams(spp=16, rfilter="box"))
    trace_bench(f"stress_{ninst}x100k", sc, d)
if "inst" in which:
    ninst = int(os.environ.get("STRESS_INSTANCES", "100"))
    for inst in (True, False):
        d = stress_scene(ninst, width=1024, height=1024, instanced=inst)
        if not inst:
            for m in d.meshes:
                if m.name.startswith("inst"):
                    m.bsdf = d.meshes[0].bsdf
        render_rate(f"stress_{ninst}x100k/" + ("instanced" if inst else "flattened"), d, RenderParams(spp=16, rfilter="box"))
if "smoke" in which:
    # config 4: 128^3 heterogeneous medium (Woodcock), isotropic phase, volpath, 512x512
    d = smoke_scene(512, 512, res=128)
    for smp in ("independent", "sobol"):
        render_rate("smoke_128/" + smp, d, RenderParams(spp=64, rfilter="gaussian", sampler=smp, integrator="volpath"), pool_size=1 << 20)
    render_rate("smoke_128/pool4M", d, RenderParams(spp=256, rfilter="gaussian", sampler="independent", integrator="volpath"))
    render_rate("smoke_128/parity_build", d, RenderParams(spp=16, rfilter="gaussian", sampler="independent", integrator="volpath"), parity=True)
    if os.environ.get("SMOKE_ORACLE", "1") == "1":  # CPU restatement on the host cores, bounded sample
        from oracle import oracle_api as O
        d2 = smoke_scene(256, 256, res=128)
        o = O.OracleScene(d2)
        rp = RenderParams(spp=16, rfilter="gaussian", sampler="independent", integrator="volpath")
        t = time.time(); _, so = o.render(rp); dt = time.time() - t
        print(json.dumps(dict(scene="smoke_128/cpu_oracle", res=256, spp=16, threads=os.cpu_count(), msamples_s=round(so["samples"] / dt / 1e6, 2), seconds=round(dt, 2))), flush=True)
