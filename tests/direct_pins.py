"""Test infrastructure of the `direct` integrator (src/integrators/direct/direct.cpp).

* `DirectOracle`: the oracle scene (oracle/oracle_api.py) rendered by tests/orc_direct.cpp -- MIDirectIntegrator::Li restated on the
  oracle, compiled together with oracle/mts_oracle.cpp into a library in the temporary directory (rebuilt when a source changes).
* `image_cases_direct()`: the image-level pins of tests/golden/path_ref_direct.npz.
* `python tests/direct_pins.py`: writes that fixture with the reference's own MIDirectIntegrator inside the renderer that
  oracle/path_ref_shim.cpp assembles from the reference's sources (tests/direct_ref_shim.cpp).  Needs the reference tree and the objects
  `make -C oracle` leaves in oracle/_build/pathref.
"""
import ctypes as C
import dataclasses
import hashlib
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
ORACLE = os.path.join(ROOT, "oracle")
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from oracle import oracle_api as O  # noqa: E402

CXX = os.environ.get("CXX", "g++")
# the oracle's flags (oracle/Makefile CXXFLAGS): IEEE-strict, no contraction
ORACLE_FLAGS = ["-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-pthread", "-Wall", "-Wno-unused-function"]
ORACLE_SOURCES = [os.path.join(HERE, f) for f in ("orc_direct.cpp", "orc_direct_sampler.h")] + \
                 [os.path.join(ORACLE, f) for f in ("mts_oracle.cpp", "orc_math.h", "orc_sampler.h", "orc_accel.h", "orc_bsdf.h", "orc_medium.h",
                                                    "orc_texture.h", "orc_envmap.h")]
_LIB = None


def _digest(paths, extra=""):
    h = hashlib.sha1(extra.encode())
    for p in paths:
        with open(p, "rb") as f:
            h.update(f.read())
    return h.hexdigest()[:16]


def build_oracle():
    """Path of the compiled oracle of `direct` (a library per source state, in the temporary directory)."""
    out = os.path.join(tempfile.gettempdir(), f"b2_orc_direct_{_digest(ORACLE_SOURCES, ' '.join(ORACLE_FLAGS))}.so")
    if not os.path.exists(out):
        tmp = f"{out}.{os.getpid()}"
        subprocess.check_call([CXX] + ORACLE_FLAGS + ["-I", ORACLE, "-shared", "-o", tmp, os.path.join(HERE, "orc_direct.cpp")])
        os.replace(tmp, out)
    return out


def lib():
    global _LIB
    if _LIB is None:
        L = C.CDLL(build_oracle())
        for name, t in (("orc_scene_new", C.c_void_p), ("orc_add_bsdf", C.c_int), ("orc_add_mesh", C.c_int), ("orc_add_medium", C.c_int),
                        ("orc_add_texture", C.c_int), ("orc_tea", C.c_uint64), ("orc_bsdf_type", C.c_uint32), ("orc_hardware_threads", C.c_int),
                        ("orcd_render", C.c_int)):
            getattr(L, name).restype = t
        _LIB = L
    return _LIB


class DirectOracle(O.OracleScene):
    """An oracle scene whose library also renders `direct` (RenderParams.integrator == "direct"); `path` / `volpath` as OracleScene."""

    def __init__(self, desc, **kw):
        saved = O._LIB
        O._LIB = lib()      # the scene lives in this library (it holds the whole oracle)
        try:
            super().__init__(desc, **kw)
        finally:
            O._LIB = saved

    def render(self, rp, threads=0, per_sample=False):
        if rp.integrator != "direct":
            return super().render(rp, threads, per_sample=per_sample)
        p = O.make_params(dataclasses.replace(rp, integrator="path"), threads)
        film = np.zeros((self.H, self.W, 5), np.float32)
        st = O.OrcStats()
        hi = rp.sample_hi if rp.sample_hi > 0 else rp.spp
        ps = np.zeros((self.H, self.W, hi - rp.sample_lo, 4), np.float32) if per_sample else None
        rc = self.L.orcd_render(self.h, C.byref(p), rp.emitter_samples, rp.bsdf_samples, O._p(film), C.byref(st), O._p(ps) if per_sample else None)
        assert rc == 0, "orcd_render: invalid counts or sampler"
        return (film, st.as_dict(), ps) if per_sample else (film, st.as_dict())


def image_cases_direct():
    """(name, SceneDesc, RenderParams) of the image-level pins: sample counts (1, 1), (4, 2), (3, 0), (0, 2), (5, 3) on both samplers and
    both filters (counts above 1 read the samplers' 2-D arrays), thin lenses with two arrays and with one (the regular draw after the
    aperture sample jumps past the array range), strictNormals + hideEmitters, a rough dielectric, a coating and a delta-only BSDF, a
    constant emitter next to an area light, an environment map (filtered look-ups on camera misses), bitmap textures (filtered at every
    shading point), instances, the smoke scene (null medium boundaries) and a crop window."""
    import ref_pins
    from bsdf_configs import configs
    from mitsuba_b200.scene import Bsdf, EnvMap, RenderParams, cornell_box, material_ball, smoke_scene, textured_scene
    cf = configs()
    D = lambda **k: RenderParams(integrator="direct", **k)
    yield "direct_cbox_11_sobol_box", cornell_box(40, 40), D(spp=8, sampler="sobol", rfilter="box")
    yield "direct_cbox_42_sobol_gaussian", cornell_box(40, 32), D(spp=4, sampler="sobol", rfilter="gaussian", emitter_samples=4, bsdf_samples=2)
    yield "direct_cbox_30_counter_box", cornell_box(32, 32), D(spp=4, sampler="independent", rfilter="box", emitter_samples=3, bsdf_samples=0)
    yield "direct_cbox_02_counter_gaussian", cornell_box(32, 32), D(spp=4, sampler="independent", rfilter="gaussian", emitter_samples=0, bsdf_samples=2)
    yield "direct_cbox_42_counter_seed", cornell_box(32, 32), D(spp=4, sampler="independent", rfilter="box", emitter_samples=4, bsdf_samples=2, seed=11)
    yield "direct_cbox_53_sobol_seed", cornell_box(24, 24), D(spp=3, sampler="sobol", rfilter="gaussian", seed=5, emitter_samples=5, bsdf_samples=3)
    d = cornell_box(36, 36)
    d.camera = dataclasses.replace(d.camera, aperture_radius=25.0, focus_distance=1100.0)
    yield "direct_thinlens_42_sobol", d, D(spp=4, sampler="sobol", rfilter="gaussian", emitter_samples=4, bsdf_samples=2, seed=3)
    yield "direct_thinlens_23_counter", d, D(spp=4, sampler="independent", rfilter="box", emitter_samples=2, bsdf_samples=3)
    yield "direct_thinlens_13_sobol", d, D(spp=4, sampler="sobol", rfilter="box", emitter_samples=1, bsdf_samples=3)
    yield "direct_thinlens_31_counter", d, D(spp=4, sampler="independent", rfilter="gaussian", emitter_samples=3, bsdf_samples=1)
    d = cornell_box(24, 20)
    d.camera = dataclasses.replace(d.camera, aperture_radius=30.0, focus_distance=1000.0)
    yield "direct_thinlens_15_sobol", d, D(spp=2, sampler="sobol", rfilter="box", emitter_samples=1, bsdf_samples=5)
    yield "direct_thinlens_51_counter", d, D(spp=2, sampler="independent", rfilter="gaussian", emitter_samples=5, bsdf_samples=1)
    yield "direct_cbox_strict_hidden", cornell_box(32, 32), D(spp=4, sampler="sobol", rfilter="box", strict_normals=True, hide_emitters=True,
                                                               emitter_samples=2, bsdf_samples=2)
    for name in ("roughdielectric_beckmann", "coating_diffuse", "dielectric"):
        yield "direct_ball_" + name, material_ball(cf[name], 36, 36, n_theta=16, n_phi=32), D(spp=4, sampler="sobol", rfilter="gaussian",
                                                                                               emitter_samples=2, bsdf_samples=3)
    d = cornell_box(36, 36)
    d.meshes = [m for i, m in enumerate(d.meshes) if i != 1]   # open the box: the environment is seen and sampled
    d.env_radiance = (0.4, 0.6, 1.0); d.env_sampling_weight = 2.0
    yield "direct_env_plus_area", d, D(spp=4, sampler="sobol", rfilter="box", emitter_samples=2, bsdf_samples=2)
    gold = Bsdf("roughconductor", distribution="ggx", alpha_u=0.2, alpha_v=0.2, eta=(0.2004, 0.9240, 1.1022), k=(3.9129, 2.4528, 2.1421))
    d = material_ball(gold, 36, 36, n_theta=16, n_phi=32)
    d.meshes = [m for m in d.meshes if m.radiance is None]
    d.envmap = EnvMap(pixels=ref_pins.sky_image(), scale=1.5, to_world=ref_pins.envmap_rotation())
    yield "direct_envmap_ball", d, D(spp=4, sampler="sobol", rfilter="gaussian", emitter_samples=3, bsdf_samples=2)
    yield "direct_tex_ewa", textured_scene(36, 36, filter_type="ewa", tex_res=32, n_theta=12, n_phi=24), D(spp=4, sampler="sobol", rfilter="gaussian",
                                                                                                            emitter_samples=2, bsdf_samples=2)
    inst = {n: d for n, d, _ in ref_pins.image_cases_ext()}["instances_sobol"]
    yield "direct_instances", inst, D(spp=4, sampler="sobol", rfilter="box", emitter_samples=2, bsdf_samples=1)
    yield "direct_smoke_null", smoke_scene(32, 32, res=8, scale=4.0), D(spp=4, sampler="independent", rfilter="gaussian")
    d = cornell_box(96, 64)
    d.camera = dataclasses.replace(d.camera, crop=(17, 9, 43, 33))
    yield "direct_crop_sobol", d, D(spp=4, sampler="sobol", rfilter="gaussian", emitter_samples=2, bsdf_samples=4)


# ---- fixture generation (reference tree present) ----------------------------------------------------------------------------------
REF = os.environ.get("MTS_REFERENCE", "/root/reference")
# oracle/Makefile PATHREF_FLAGS: the flags the assembled reference renderer's objects were compiled with
PATHREF_FLAGS = ["-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fpermissive", "-w", "-DSINGLE_PRECISION", "-DSPECTRUM_SAMPLES=3",
                 "-include", "unistd.h", "-I" + os.path.join(ORACLE, "shim_core"), "-I" + os.path.join(REF, "include"),
                 "-include", "mitsuba/render/shape.h", "-include", "mitsuba/core/half.h", "-DMTS_NO_STATISTICS",
                 "-I" + os.path.join(REF, "src", "samplers"), "-I" + os.path.join(REF, "src", "shapes"), "-I" + ORACLE, "-I" + HERE]


def build_reference(workdir):
    """The assembled reference renderer + MIDirectIntegrator + tests/direct_ref_shim.cpp as one library in `workdir`."""
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else CXX   # the system compiler, as oracle/Makefile REFCXX
    objdir = os.path.join(ORACLE, "_build", "pathref")
    objs = sorted(os.path.join(objdir, f) for f in os.listdir(objdir) if f.endswith(".o") and f != "zz_shim.o")
    d = os.path.join(workdir, "p_direct.o")
    subprocess.check_call([cxx] + PATHREF_FLAGS + ["-DCreateInstance=CreateInstance_direct", "-DGetDescription=GetDescription_direct", "-c",
                                                   os.path.join(REF, "src", "integrators", "direct", "direct.cpp"), "-o", d])
    s = os.path.join(workdir, "zz_direct_shim.o")
    subprocess.check_call([cxx] + PATHREF_FLAGS + ["-c", os.path.join(HERE, "direct_ref_shim.cpp"), "-o", s])
    so = os.path.join(workdir, "libdirectref.so")
    subprocess.check_call([cxx, "-shared", "-o", so] + objs + [d, s, "-lz"])
    return so


def reference_render_direct(lib, desc, rp):
    """Film (H, W, 5), sampleToCamera, instance inverses and the envmap's inverse of one case, rendered by the reference's `direct`."""
    import ref_pins
    h = ref_pins.reference_scene(lib, desc, dataclasses.replace(rp, integrator="path"))
    cam = desc.camera
    fw, fh = cam.film_size()
    lib.pathref_use_direct(h, {"sobol": 0, "independent": 2}[rp.sampler], fw, rp.spp, C.c_uint64(rp.seed), rp.emitter_samples, rp.bsdf_samples,
                           int(rp.strict_normals), int(rp.hide_emitters))
    film = np.zeros((fh, fw, 5), np.float32)
    lib.pathref_render(h, O._p(film))
    s2c = np.zeros((4, 4), np.float32)
    lib.pathref_sample_to_camera(h, O._p(s2c))
    return film, s2c, ref_pins.reference_instance_inverses(lib, desc), ref_pins.reference_envmap_inverse(lib, desc)


def generate():
    sys.path.insert(0, HERE)
    with tempfile.TemporaryDirectory() as wd:
        lib = C.CDLL(build_reference(wd))
        out = {}
        for name, desc, rp in image_cases_direct():
            film, s2c, inv, env = reference_render_direct(lib, desc, rp)
            out[name + "/film"], out[name + "/s2c"] = film, s2c
            if inv:
                out[name + "/instance_inverses"] = np.stack(inv)
            if env is not None:
                out[name + "/env_to_local"] = env
        np.savez_compressed(os.path.join(HERE, "golden", "path_ref_direct.npz"), **out)
        print("path_ref_direct.npz:", sum(k.endswith("/film") for k in out), "images")


if __name__ == "__main__":
    generate()
