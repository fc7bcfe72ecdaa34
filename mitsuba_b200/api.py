"""ctypes binding of the C-ABI (include/b2mts.h) -- the Python host side used by tests, bench.py and
the multi-GPU driver.  Everything here calls libb2mts.so; there is no Python or CPU compute fallback:
when the library (or a GPU) is missing the calls raise.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from .scene import RenderParams, SceneDesc

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIBPATH = os.environ.get("B2MTS_LIB", os.path.join(_HERE, "libb2mts.so"))  # B2MTS_LIB: A/B builds of the same ABI
_LIB = None


class B2Error(RuntimeError):
    pass


class b2_material_desc(C.Structure):
    _fields_ = [("type", C.c_int32), ("distr", C.c_int32), ("sample_visible", C.c_int32), ("nested", C.c_int32),
                ("alpha_u", C.c_float), ("alpha_v", C.c_float), ("eta", C.c_float), ("thickness", C.c_float),
                ("reflectance", C.c_float * 3), ("transmittance", C.c_float * 3), ("eta_c", C.c_float * 3),
                ("k_c", C.c_float * 3), ("sigma_a", C.c_float * 3), ("nested2", C.c_int32), ("diffuse_reflectance", C.c_float * 3),
                ("fdr_int", C.c_float), ("fdr_ext", C.c_float), ("spec_sampling_weight", C.c_float), ("nonlinear", C.c_int32),
                ("reflectance_texture", C.c_int32)]


class b2_texture_desc(C.Structure):
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("channels", C.c_int32), ("filter_type", C.c_int32),
                ("wrap_u", C.c_int32), ("wrap_v", C.c_int32), ("max_anisotropy", C.c_float), ("uoffset", C.c_float),
                ("voffset", C.c_float), ("uscale", C.c_float), ("vscale", C.c_float), ("reserved", C.c_uint32),
                ("pixels", C.POINTER(C.c_float))]


class b2_render_params(C.Structure):
    _fields_ = [("spp", C.c_int32), ("sampler", C.c_int32), ("seed", C.c_uint64), ("max_depth", C.c_int32),
                ("rr_depth", C.c_int32), ("strict_normals", C.c_int32), ("hide_emitters", C.c_int32),
                ("rfilter", C.c_int32), ("rfilter_param", C.c_float), ("sample_lo", C.c_int32), ("sample_hi", C.c_int32),
                ("parity_mode", C.c_int32), ("pool_size", C.c_int32), ("film_on_device", C.c_int32), ("flags", C.c_int32),
                ("integrator", C.c_int32), ("emitter_samples", C.c_int16), ("bsdf_samples", C.c_int16)]


class b2_medium_desc(C.Structure):
    _fields_ = [("type", C.c_int32), ("phase", C.c_int32), ("g", C.c_float), ("sigma_a", C.c_float * 3), ("sigma_s", C.c_float * 3),
                ("strategy", C.c_int32), ("sampling_density", C.c_float), ("medium_sampling_weight", C.c_float), ("scale", C.c_float),
                ("albedo", C.c_float * 3), ("res", C.c_int32 * 3), ("world_to_grid", C.c_float * 12), ("aabb_min", C.c_float * 3),
                ("aabb_max", C.c_float * 3), ("density", C.POINTER(C.c_float))]


INTEGRATORS = {"path": 0, "volpath": 1, "direct": 2}


class b2_stats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("samples", "rays", "shadow_rays", "path_length_sum", "bad_samples", "dim_overflow",
                                          "node_visits", "prim_tests", "iterations", "kernel_launches")] + \
               [(n, C.c_float) for n in ("ms_total", "ms_generate", "ms_extend", "ms_shade", "ms_occluded", "ms_film")] + \
               [(n, C.c_uint64) for n in ("n_triangles", "n_bvh_nodes", "n_generate", "n_extend", "n_shade", "n_occluded",
                                          "bytes_uploaded", "pool_size", "unoccluded_shadow_rays", "bvh_node_bytes")] + \
               [("accel_build_ms", C.c_float), ("accel_build_mode", C.c_int32)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


EXPORTS = ["b2_context_create", "b2_context_destroy", "b2_last_error", "b2_scene_create", "b2_scene_destroy",
           "b2_scene_set_camera", "b2_scene_set_crop", "b2_scene_set_thinlens", "b2_scene_get_sample_to_camera", "b2_scene_film_size", "b2_scene_add_material", "b2_scene_add_area_emitter",
           "b2_scene_add_mesh", "b2_scene_add_shapegroup", "b2_scene_set_mesh_group", "b2_scene_add_instance", "b2_scene_add_constant_emitter", "b2_scene_add_envmap_emitter", "b2_envmap_probe", "b2_load_image", "b2_spectrum_to_rgb", "b2_scene_add_medium", "b2_scene_set_mesh_media", "b2_medium_probe", "b2_scene_add_texture", "b2_texture_eval", "b2_texture_partials", "b2_texture_level", "b2_mipmap_level", "b2_scene_commit", "b2_render", "b2_cancel", "b2_film_develop", "b2_get_stats", "b2_get_pixel_stats", "b2_get_path_traces", "b2_trace",
           "b2_trace_device", "b2_bsdf_eval", "b2_bsdf_sample", "b2_sample_emitter_direct", "b2_sampler_stream",
           "b2_camera_rays", "b2_splat", "b2_get_triaccel", "b2_load_xml", "b2_version", "b2_device_count",
           "b2_scene_set_accel_build", "b2_context_set_accel_build", "b2_scene_get_accel"]

ACCEL_BUILDS = {"host": 0, "device": 1}


def _accel_mode(name):
    if name not in ACCEL_BUILDS:
        raise B2Error(f"accel_build must be one of {sorted(ACCEL_BUILDS)}, not {name!r}")
    return ACCEL_BUILDS[name]


def lib():
    """Load libb2mts.so (built in-tree by mitsuba_b200.build).  Raises if it is missing: no fallback."""
    global _LIB
    if _LIB is None:
        if not os.path.exists(_LIBPATH):
            raise B2Error(f"{_LIBPATH} not built: run `python -m mitsuba_b200.build` (there is no CPU fallback)")
        L = C.CDLL(_LIBPATH)
        L.b2_last_error.restype = C.c_char_p
        L.b2_last_error.argtypes = [C.c_void_p]
        L.b2_version.restype = C.c_char_p
        for name in ("b2_scene_add_material", "b2_scene_add_area_emitter", "b2_scene_add_mesh", "b2_scene_add_medium", "b2_scene_add_constant_emitter", "b2_scene_add_envmap_emitter"):
            getattr(L, name).restype = C.c_int
        _LIB = L
    return _LIB


def spectrum_to_rgb(wavelengths, values, zero_extend=True):
    """(wavelength nm, value) samples -> linear RGB as the scene file's <spectrum> tags are converted (b2_spectrum_to_rgb; host-only)."""
    L = lib()
    w = np.ascontiguousarray(wavelengths, np.float32); v = np.ascontiguousarray(values, np.float32)
    rgb = np.zeros(3, np.float32)
    err = C.create_string_buffer(1024)
    if L.b2_spectrum_to_rgb(w.ctypes.data_as(C.POINTER(C.c_float)), v.ctypes.data_as(C.POINTER(C.c_float)), C.c_int(len(w)), C.c_int(int(zero_extend)),
                            rgb.ctypes.data_as(C.POINTER(C.c_float)), err, 1024):
        raise B2Error(err.value.decode(errors="replace"))
    return rgb


def load_image(path, gamma=0.0):
    """Decode an image file with the scene-file front end's readers (b2_load_image; host-only): OpenEXR scan-line, Radiance RGBE, PFM,
    8-bit PPM -> float32 (H, W, C) linear, top row first."""
    L = lib()
    w, h, c = C.c_int(), C.c_int(), C.c_int()
    err = C.create_string_buffer(1024)
    if L.b2_load_image(str(path).encode(), C.c_float(gamma), C.byref(w), C.byref(h), C.byref(c), None, err, 1024):
        raise B2Error(err.value.decode(errors="replace"))
    out = np.zeros((h.value, w.value, c.value), np.float32)
    if L.b2_load_image(str(path).encode(), C.c_float(gamma), C.byref(w), C.byref(h), C.byref(c), out.ctypes.data_as(C.POINTER(C.c_float)), err, 1024):
        raise B2Error(err.value.decode(errors="replace"))
    return out


def _p(a, t=C.c_float):
    return a.ctypes.data_as(C.POINTER(t)) if a is not None else None


SAMPLERS = {"sobol": 0, "independent": 2}
RFILTERS = {"box": 0, "gaussian": 1}


def make_params(rp: RenderParams, parity=False, pool_size=0, film_on_device=False, flags=0) -> b2_render_params:
    p = b2_render_params()
    p.spp, p.sampler, p.seed = rp.spp, SAMPLERS[rp.sampler], rp.seed
    p.max_depth, p.rr_depth = rp.max_depth, rp.rr_depth
    p.strict_normals, p.hide_emitters = int(rp.strict_normals), int(rp.hide_emitters)
    p.rfilter, p.rfilter_param = RFILTERS[rp.rfilter], rp.rfilter_param
    p.sample_lo, p.sample_hi = rp.sample_lo, rp.sample_hi
    p.parity_mode, p.pool_size, p.film_on_device, p.flags = int(parity), pool_size, int(film_on_device), flags
    p.integrator = INTEGRATORS[getattr(rp, "integrator", "path")]
    for name in ("emitter_samples", "bsdf_samples"):   # int16 fields: an out-of-range count must not wrap into a valid one
        v = int(getattr(rp, name, 1))
        if not -32768 <= v <= 32767:
            raise B2Error(f"{name} out of range: {v}")
        setattr(p, name, v)
    return p


def params_to_render_params(p: b2_render_params) -> RenderParams:
    inv_s = {v: k for k, v in SAMPLERS.items()}
    inv_f = {v: k for k, v in RFILTERS.items()}
    return RenderParams(spp=p.spp, sampler=inv_s[p.sampler], seed=p.seed, max_depth=p.max_depth, rr_depth=p.rr_depth,
                        strict_normals=bool(p.strict_normals), hide_emitters=bool(p.hide_emitters), rfilter=inv_f[p.rfilter],
                        rfilter_param=p.rfilter_param, sample_lo=p.sample_lo, sample_hi=p.sample_hi,
                        integrator={v: k for k, v in INTEGRATORS.items()}[p.integrator],
                        emitter_samples=p.emitter_samples, bsdf_samples=p.bsdf_samples)


class Context:
    """One per GPU / rank (b2_context_create)."""

    def __init__(self, device: int = 0):
        self.L = lib()
        self.h = C.c_void_p()
        rc = self.L.b2_context_create(C.c_int(device), C.byref(self.h))
        if rc:
            raise B2Error(f"b2_context_create({device}) failed [{rc}]: {self.L.b2_last_error(None).decode()}")
        self.device = device

    def err(self):
        return self.L.b2_last_error(self.h).decode()

    def close(self):
        if self.h:
            self.L.b2_context_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def splat(self, W, H, kind, param, pos, val):
        pos = np.ascontiguousarray(pos, np.float32).reshape(-1, 2)
        val = np.ascontiguousarray(val, np.float32).reshape(-1, 4)
        film = np.zeros((H, W, 5), np.float32)
        rc = self.L.b2_splat(self.h, C.c_int(W), C.c_int(H), C.c_int(RFILTERS[kind]), C.c_float(param), C.c_uint64(len(pos)),
                             _p(pos), _p(val), _p(film))
        if rc:
            raise B2Error(self.err())
        return film

    def set_accel_build(self, accel_build):
        """Builder ("host" | "device") of the scenes created on this context from now on (b2_context_set_accel_build)."""
        if self.L.b2_context_set_accel_build(self.h, C.c_int(_accel_mode(accel_build))):
            raise B2Error(self.err())

    def load_xml(self, path, defines=(), accel_build=None):
        """accel_build: "host" | "device" sets the context's default builder first (it stays set for later scenes)."""
        if accel_build is not None:
            self.set_accel_build(accel_build)
        hs = C.c_void_p()
        p = b2_render_params()
        arr = (C.c_char_p * max(1, len(defines)))(*[d.encode() for d in defines])
        rc = self.L.b2_load_xml(self.h, path.encode(), arr, C.c_int(len(defines)), C.byref(hs), C.byref(p))
        if rc:
            raise B2Error(f"b2_load_xml failed [{rc}]: {self.err()}")
        sc = Scene.__new__(Scene)
        sc.ctx, sc.L, sc.h = self, self.L, hs
        W = C.c_int(); H = C.c_int()
        self.L.b2_scene_film_size(hs, C.byref(W), C.byref(H))
        sc.W, sc.H = W.value, H.value
        sc.material_ids = None
        return sc, params_to_render_params(p)


class Scene:
    """Device scene built from a SceneDesc through the C-ABI."""

    def __init__(self, ctx: Context, desc: SceneDesc, accel_build=None):
        """accel_build: "host" | "device" acceleration-structure builder; None = the context's default (host unless changed)."""
        self.ctx, self.L = ctx, ctx.L
        self.h = C.c_void_p()
        self._ck(self.L.b2_scene_create(ctx.h, C.byref(self.h)))
        if accel_build is not None:
            self._ck(self.L.b2_scene_set_accel_build(self.h, C.c_int(_accel_mode(accel_build))))
        cam = desc.camera
        self.W, self.H = cam.film_size()
        c2w = np.ascontiguousarray(cam.to_world, np.float32)
        self._ck(self.L.b2_scene_set_camera(self.h, _p(c2w), C.c_float(cam.xfov()), C.c_float(cam.near), C.c_float(cam.far),
                                            C.c_int(cam.width), C.c_int(cam.height)))
        if getattr(cam, "crop", None):
            self._ck(self.L.b2_scene_set_crop(self.h, *[C.c_int(int(v)) for v in cam.crop]))
        if getattr(cam, "aperture_radius", 0.0) > 0:
            self._ck(self.L.b2_scene_set_thinlens(self.h, C.c_float(cam.aperture_radius), C.c_float(cam.focus_distance if cam.focus_distance > 0 else cam.far)))
        flat, ids = desc.flat_bsdfs()
        self.flat_bsdfs = flat
        self.material_ids = ids
        self.flat_textures = desc.flat_textures()
        for d in self.flat_textures:  # bitmap textures first: materials refer to them by id
            t = b2_texture_desc()
            t.width, t.height, t.channels, t.filter_type = d["width"], d["height"], d["channels"], d["filterType"]
            t.wrap_u, t.wrap_v, t.max_anisotropy = d["wrapU"], d["wrapV"], d["maxAnisotropy"]
            t.uoffset, t.voffset, t.uscale, t.vscale = d["uoffset"], d["voffset"], d["uscale"], d["vscale"]
            t.pixels = d["pixels"].ctypes.data_as(C.POINTER(C.c_float))
            if self.L.b2_scene_add_texture(self.h, C.byref(t)) < 0:
                raise B2Error(ctx.err())
        for d in flat:
            m = b2_material_desc()
            m.reflectance_texture = d.get("texture", -1) + 1
            m.type, m.distr, m.sample_visible, m.nested = d["type"], d["distr"], d["sampleVisible"], d["nested"]
            m.alpha_u, m.alpha_v, m.eta, m.thickness = d["alphaU"], d["alphaV"], d["eta"], d["thickness"]
            for k, src in (("reflectance", "reflectance"), ("transmittance", "transmittance"), ("eta_c", "etaC"), ("k_c", "kC"), ("sigma_a", "sigmaA"),
                           ("diffuse_reflectance", "diffuseReflectance")):
                for j in range(3):
                    getattr(m, k)[j] = d[src][j]
            m.nested2, m.fdr_int, m.fdr_ext, m.spec_sampling_weight, m.nonlinear = d["nested2"], d["fdrInt"], d["fdrExt"], d["specSamplingWeight"], d["nonlinear"]
            if self.L.b2_scene_add_material(self.h, C.byref(m)) < 0:
                raise B2Error(ctx.err())
        media, media_ids = desc.flat_media()
        self.flat_media = [md.flat() for md in media]
        for d in self.flat_media:
            m = b2_medium_desc()
            m.type, m.phase, m.g, m.strategy = d["type"], d["phase"], d["g"], d["strategy"]
            m.sampling_density, m.medium_sampling_weight, m.scale = d["samplingDensity"], d["mediumSamplingWeight"], d["scale"]
            for k, src in (("sigma_a", "sigmaA"), ("sigma_s", "sigmaS"), ("albedo", "albedo"), ("aabb_min", "aabbMin"), ("aabb_max", "aabbMax")):
                for j in range(3):
                    getattr(m, k)[j] = d[src][j]
            for j in range(3):
                m.res[j] = d["res"][j]
            for j in range(12):
                m.world_to_grid[j] = d["worldToGrid"][j]
            m.density = d["density"].ctypes.data_as(C.POINTER(C.c_float)) if d["density"] is not None else None
            if self.L.b2_scene_add_medium(self.h, C.byref(m)) < 0:
                raise B2Error(ctx.err())
        for _ in range(desc.n_groups()):
            self.L.b2_scene_add_shapegroup(self.h)
        for mesh, bid in zip(desc.meshes, ids):
            eid = -1
            if mesh.radiance is not None:
                rad = np.asarray(mesh.radiance, np.float32)
                eid = self.L.b2_scene_add_area_emitter(self.h, _p(rad), C.c_float(mesh.sampling_weight))
                if eid < 0:
                    raise B2Error(ctx.err())
            P = np.ascontiguousarray(mesh.P, np.float32)
            N = np.ascontiguousarray(mesh.N, np.float32) if mesh.N is not None else None
            UV = np.ascontiguousarray(mesh.UV, np.float32) if mesh.UV is not None else None
            I = np.ascontiguousarray(mesh.idx, np.uint32)
            mid = self.L.b2_scene_add_mesh(self.h, _p(P), _p(N), _p(UV), C.c_uint32(len(P)), _p(I, C.c_uint32), C.c_uint32(len(I)),
                                           C.c_int(bid), C.c_int(eid))
            if mid < 0:
                raise B2Error(ctx.err())
            if mesh.group >= 0:
                self._ck(self.L.b2_scene_set_mesh_group(self.h, C.c_int(mid), C.c_int(mesh.group)))
        for inst in desc.instances:
            M64 = np.asarray(inst.to_world, np.float64)
            M, Minv = np.ascontiguousarray(M64, np.float32), np.ascontiguousarray(np.linalg.inv(M64), np.float32)
            if self.L.b2_scene_add_instance(self.h, C.c_int(inst.group), _p(M), _p(Minv)) < 0:
                raise B2Error(ctx.err())
        if getattr(desc, "env_radiance", None) is not None:
            rad = np.asarray(desc.env_radiance, np.float32)
            if self.L.b2_scene_add_constant_emitter(self.h, _p(rad), C.c_float(desc.env_sampling_weight)) < 0:
                raise B2Error(ctx.err())
        if getattr(desc, "envmap", None) is not None:
            em = desc.envmap
            px = np.ascontiguousarray(em.pixels, np.float32)
            if px.ndim != 3 or px.shape[2] != 3:
                raise B2Error("envmap pixels must be (H, W, 3) linear float RGB")
            M, Minv = em.matrices()
            ident = em.to_world is None
            if self.L.b2_scene_add_envmap_emitter(self.h, C.c_int(px.shape[1]), C.c_int(px.shape[0]), _p(px), C.c_float(em.scale),
                                                  None if ident else _p(M), None if ident else _p(Minv), C.c_float(em.sampling_weight)) < 0:
                raise B2Error(ctx.err())
        for i, (mi, me) in enumerate(media_ids):
            if mi >= 0 or me >= 0:
                self._ck(self.L.b2_scene_set_mesh_media(self.h, C.c_int(i), C.c_int(mi), C.c_int(me)))
        self._ck(self.L.b2_scene_commit(self.h))

    def _ck(self, rc):
        if rc:
            raise B2Error(f"[{rc}] {self.ctx.err()}")

    def close(self):
        if getattr(self, "h", None):
            self.L.b2_scene_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def sample_to_camera(self):
        out = np.zeros(16, np.float32)
        self._ck(self.L.b2_scene_get_sample_to_camera(self.h, _p(out)))
        return out.reshape(4, 4)

    def stats(self):
        st = b2_stats()
        self.L.b2_get_stats(self.h, C.byref(st))
        return st.as_dict()

    def pixel_stats(self):
        """(H, W) uint64 of the last render(flags=32): (sum of squared path lengths << 32) | sum of path lengths per pixel."""
        out = np.zeros((self.H, self.W), np.uint64)
        self._ck(self.L.b2_get_pixel_stats(self.h, out.ctypes.data_as(C.POINTER(C.c_uint64))))
        return out

    def path_traces(self, n_samples):
        """(H, W, n_samples) uint64 event traces of the last render(flags=64), one byte per bounce (include/b2mts.h)."""
        out = np.zeros((self.H, self.W, n_samples), np.uint64)
        self._ck(self.L.b2_get_path_traces(self.h, C.c_uint64(out.size), out.ctypes.data_as(C.POINTER(C.c_uint64))))
        return out

    def accel_arrays(self):
        """The committed acceleration arrays as they sit in device memory (b2_scene_get_accel): binary nodes and 8-wide nodes as raw
        bytes (64 / 80 bytes per node), leaf-ordered prim ids as uint32."""
        out = {}
        for key, which in (("nodes", 0), ("nodes8", 1), ("leaf_prims", 2)):
            n = C.c_uint64()
            self._ck(self.L.b2_scene_get_accel(self.h, C.c_int(which), None, C.byref(n)))
            buf = np.zeros(n.value, np.uint8)
            self._ck(self.L.b2_scene_get_accel(self.h, C.c_int(which), buf.ctypes.data_as(C.c_void_p), C.byref(n)))
            out[key] = buf.tobytes() if key != "leaf_prims" else buf.view(np.uint32)
        return out

    def triaccel(self):
        n = self.stats()["n_triangles"]
        out = np.zeros((n, 12), np.float32)
        self._ck(self.L.b2_get_triaccel(self.h, _p(out)))
        return out

    def render(self, rp: RenderParams, parity=False, pool_size=0, flags=0, film=None, width=None, height=None):
        """Returns (film H x W x 5 float32 host array, stats).  `film`: optional torch CUDA tensor (H,W,5) to fill in place."""
        W, H = width or self.W, height or self.H
        if film is not None:
            p = make_params(rp, parity, pool_size, True, flags)
            assert film.is_cuda and film.is_contiguous() and film.numel() == W * H * 5
            self._ck(self.L.b2_render(self.h, C.byref(p), C.c_void_p(film.data_ptr())))
            return film, self.stats()
        p = make_params(rp, parity, pool_size, False, flags)
        out = np.zeros((H, W, 5), np.float32)
        self._ck(self.L.b2_render(self.h, C.byref(p), _p(out)))
        return out, self.stats()

    def trace(self, rays, mode=0, parity=True):
        rays = np.ascontiguousarray(rays, np.float32).reshape(-1, 8)
        n = len(rays)
        t = np.zeros(n, np.float32); u = np.zeros(n, np.float32); v = np.zeros(n, np.float32); prim = np.zeros(n, np.uint32)
        ms = C.c_float()
        self._ck(self.L.b2_trace(self.h, C.c_uint64(n), _p(rays), C.c_int(mode), C.c_int(int(parity)), _p(t), _p(u), _p(v),
                                 _p(prim, C.c_uint32), C.byref(ms)))
        return t, u, v, prim

    def trace_device(self, d_rays, d_out, n, mode=0, parity=False):
        """d_rays / d_out: torch CUDA float32 tensors (n*8, n*4).  Returns kernel ms."""
        ms = C.c_float()
        self._ck(self.L.b2_trace_device(self.h, C.c_uint64(n), C.c_void_p(d_rays.data_ptr()), C.c_int(mode), C.c_int(int(parity)),
                                        C.c_void_p(d_out.data_ptr()), C.byref(ms)))
        return ms.value

    def camera_rays(self, pos, parity=True):
        pos = np.ascontiguousarray(pos, np.float32).reshape(-1, 2)
        rays = np.zeros((len(pos), 8), np.float32)
        self._ck(self.L.b2_camera_rays(self.h, C.c_uint64(len(pos)), _p(pos), C.c_int(int(parity)), _p(rays)))
        return rays

    def bsdf_eval(self, mat, wi, wo, parity=True):
        wi = np.ascontiguousarray(wi, np.float32).reshape(-1, 3); wo = np.ascontiguousarray(wo, np.float32).reshape(-1, 3)
        rgb = np.zeros((len(wi), 3), np.float32); pdf = np.zeros(len(wi), np.float32)
        self._ck(self.L.b2_bsdf_eval(self.h, C.c_int(mat), C.c_uint64(len(wi)), _p(wi), _p(wo), C.c_int(int(parity)), _p(rgb), _p(pdf)))
        return rgb, pdf

    def bsdf_sample(self, mat, wi, samples, parity=True):
        wi = np.ascontiguousarray(wi, np.float32).reshape(-1, 3); samples = np.ascontiguousarray(samples, np.float32).reshape(-1, 3)
        out = np.zeros((len(wi), 10), np.float32)
        self._ck(self.L.b2_bsdf_sample(self.h, C.c_int(mat), C.c_uint64(len(wi)), _p(wi), _p(samples), C.c_int(int(parity)), _p(out)))
        return dict(wo=out[:, 0:3], weight=out[:, 3:6], pdf=out[:, 6], type=out[:, 7].astype(np.uint32), eta=out[:, 8])

    def sample_emitter_direct(self, ref, samples, parity=True):
        ref = np.ascontiguousarray(ref, np.float32).reshape(-1, 6); samples = np.ascontiguousarray(samples, np.float32).reshape(-1, 2)
        out = np.zeros((len(ref), 12), np.float32)
        self._ck(self.L.b2_sample_emitter_direct(self.h, C.c_uint64(len(ref)), _p(ref), _p(samples), C.c_int(int(parity)), _p(out)))
        return out

    def envmap_probe(self, what, data, parity=True):
        """what: 'eval' (n,3 directions) | 'eval_diff' (n,9: d, rxDirection, ryDirection) | 'pdf' (n,3 directions) (b2_envmap_probe)."""
        w = {"eval": (0, 3, 3), "eval_diff": (1, 9, 3), "pdf": (2, 3, 1)}[what]
        data = np.ascontiguousarray(data, np.float32).reshape(-1, w[1])
        out = np.zeros((len(data), w[2]), np.float32)
        self._ck(self.L.b2_envmap_probe(self.h, C.c_int(w[0]), C.c_uint64(len(data)), _p(data), C.c_int(int(parity)), _p(out)))
        return out[:, 0] if w[2] == 1 else out

    def medium_probe(self, medium, what, data, seed=0, parity=True):
        """what: 'transmittance' | 'sample_distance' | 'density' | 'phase' (b2_medium_probe)."""
        w = {"transmittance": (0, 8, 3), "sample_distance": (1, 8, 12), "density": (2, 3, 1), "phase": (3, 5, 5)}[what]
        data = np.ascontiguousarray(data, np.float32).reshape(-1, w[1])
        out = np.zeros((len(data), w[2]), np.float32)
        self._ck(self.L.b2_medium_probe(self.h, C.c_int(medium), C.c_int(w[0]), C.c_uint64(len(data)), _p(data), C.c_uint64(seed),
                                        C.c_int(int(parity)), _p(out)))
        return out[:, 0] if w[2] == 1 else out

    def texture_eval(self, tex, uv, partials=None, parity=True):
        """Texture2D::eval (b2_texture_eval): uv (n,2); partials (n,4) = dudx, dudy, dvdx, dvdy or None (no ray differentials)."""
        uv = np.ascontiguousarray(uv, np.float32).reshape(-1, 2)
        pt = np.ascontiguousarray(partials, np.float32).reshape(-1, 4) if partials is not None else None
        out = np.zeros((len(uv), 3), np.float32)
        self._ck(self.L.b2_texture_eval(self.h, C.c_int(tex), C.c_uint64(len(uv)), _p(uv), _p(pt), C.c_int(int(parity)), _p(out)))
        return out

    def texture_partials(self, pos, hits, spp, parity=True):
        """uv + uv partials of camera-ray hits (b2_texture_partials): pos (n,2) film positions, hits = (t, u, v, prim) arrays of trace()."""
        t, u, v, prim = hits
        rec = np.zeros((len(t), 6), np.float32)
        rec[:, 0:2] = np.asarray(pos, np.float32).reshape(-1, 2)
        rec[:, 2], rec[:, 3], rec[:, 4] = t, u, v
        rec[:, 5] = np.asarray(prim, np.uint32).view(np.float32)
        out = np.zeros((len(t), 6), np.float32)
        self._ck(self.L.b2_texture_partials(self.h, C.c_uint64(len(t)), _p(rec), C.c_int(spp), C.c_int(int(parity)), _p(out)))
        return out

    def texture_level(self, tex, level):
        """One level of the MIP pyramid commit built (b2_texture_level) as (h, w, channels)."""
        n, w, h = C.c_int(), C.c_int(), C.c_int()
        self._ck(self.L.b2_texture_level(self.h, C.c_int(tex), C.c_int(level), C.byref(n), C.byref(w), C.byref(h), None))
        out = np.zeros((h.value, w.value, self.flat_textures[tex]["channels"]), np.float32)
        self._ck(self.L.b2_texture_level(self.h, C.c_int(tex), C.c_int(level), C.byref(n), C.byref(w), C.byref(h), _p(out)))
        return out, n.value

    def sampler_stream(self, kind, seed, spp, px, py, sample_idx, ndim):
        out = np.zeros(ndim, np.float32)
        self._ck(self.L.b2_sampler_stream(self.h, C.c_int(SAMPLERS[kind]), C.c_uint64(seed), C.c_int(spp), C.c_int(px), C.c_int(py),
                                          C.c_int(sample_idx), C.c_int(ndim), _p(out)))
        return out


def develop(film):
    film = np.ascontiguousarray(film, np.float32)
    H, W = film.shape[:2]
    rgb = np.zeros((H, W, 3), np.float32)
    rc = lib().b2_film_develop(_p(film), C.c_int(W), C.c_int(H), _p(rgb))
    if rc:
        raise B2Error("b2_film_develop failed")
    return rgb


def device_count() -> int:
    return int(lib().b2_device_count())
