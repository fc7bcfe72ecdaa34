"""Acceleration-structure build time, host builder vs device builder, on the flattened stress scene (and optionally the instanced
config-5 scene).  Prints one JSON line.

    python scripts/accel_build_bench.py [--instances 25 100] [--reps 3] [--instanced]

Per scene and builder: accel_build_ms (host: wall time of the builds on all usable threads; device: CUDA-event time from the box upload
to the leaf-order readback) and the wall time of the whole b2_scene_commit, as median and min..max over --reps commits after one
warm-up commit; tree sizes; the card's name and power limit (read as bench.py reads them)."""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from mitsuba_b200 import api  # noqa: E402
from mitsuba_b200.scene import stress_scene  # noqa: E402


def gpu_info():
    from bench import gpu_info as info
    return info(0)


def usable_threads():
    return len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else os.cpu_count()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--instances", type=int, nargs="+", default=[25, 100])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--instanced", action="store_true", help="also the instanced config-5 scene (stress_scene(100, instanced=True))")
    args = ap.parse_args()
    ctx = api.Context(0)
    L = ctx.L
    commit = L.b2_scene_commit
    walls = []

    def timed_commit(h):   # wall time of b2_scene_commit alone (the scene description is handed over before)
        t = time.perf_counter()
        rc = commit(h)
        walls.append((time.perf_counter() - t) * 1e3)
        return rc

    L.b2_scene_commit = timed_commit
    scenes = [(f"flat{n}", lambda n=n: stress_scene(n, width=64, height=64)) for n in args.instances]
    if args.instanced:
        scenes.append(("instanced100", lambda: stress_scene(100, width=64, height=64, instanced=True)))
    out = {"gpu": gpu_info(), "host_threads": usable_threads(), "reps": args.reps, "scenes": {}}
    for name, make in scenes:
        d = make()
        rec = {"triangles": d.n_triangles()}
        for mode in ("host", "device"):
            build, wall = [], []
            for rep in range(args.reps + 1):
                walls.clear()
                sc = api.Scene(ctx, d, accel_build=mode)
                st = sc.stats()
                sc.close()
                if rep == 0:
                    rec["bvh_nodes"] = st["n_bvh_nodes"]; rec["bvh_node_bytes"] = st["bvh_node_bytes"]
                    continue   # warm-up
                build.append(st["accel_build_ms"]); wall.append(walls[-1])
            rec[mode] = {"accel_build_ms": statistics.median(build), "accel_build_ms_range": [min(build), max(build)],
                         "commit_ms": statistics.median(wall), "commit_ms_range": [min(wall), max(wall)]}
        rec["build_speedup"] = rec["host"]["accel_build_ms"] / rec["device"]["accel_build_ms"]
        rec["commit_speedup"] = rec["host"]["commit_ms"] / rec["device"]["commit_ms"]
        out["scenes"][name] = rec
        print(f"# {name}: {json.dumps(rec)}", file=sys.stderr, flush=True)
    L.b2_scene_commit = commit
    ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
