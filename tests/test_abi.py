"""The C-ABI library builds, loads and exports every symbol include/b2mts.h declares (no compute calls)."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "b2mts.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(b2_[a-z_0-9]+)\s*\(", src)))


def test_header_declares_the_boundary():
    syms = declared_symbols()
    for must in ("b2_context_create", "b2_scene_add_mesh", "b2_scene_commit", "b2_render", "b2_trace", "b2_load_xml", "b2_film_develop"):
        assert must in syms


def test_library_exports_every_declared_symbol():
    from mitsuba_b200 import api
    L = api.lib()
    missing = [s for s in declared_symbols() if not hasattr(L, s)]
    assert not missing, missing
    assert set(api.EXPORTS) <= set(declared_symbols())
    assert b"sm_90a" in L.b2_version()


def test_struct_layouts_match_header():
    from mitsuba_b200 import api
    assert ctypes.sizeof(api.b2_material_desc) == 4 * 4 + 4 * 4 + 15 * 4 + 9 * 4 and api.b2_material_desc.nested2.offset == 92
    assert api.b2_material_desc.reflectance_texture.offset == 124
    assert ctypes.sizeof(api.b2_texture_desc) == 56 and api.b2_texture_desc.pixels.offset == 48
    assert ctypes.sizeof(api.b2_render_params) == 72
    assert api.b2_render_params.seed.offset == 8 and api.b2_render_params.flags.offset == 60 and api.b2_render_params.integrator.offset == 64
    # b2_medium_desc: 37 four-byte fields (148 B), padding, one pointer
    assert api.b2_medium_desc.aabb_max.offset == 136 and api.b2_medium_desc.density.offset == 152 and ctypes.sizeof(api.b2_medium_desc) == 160


def test_no_cpu_fallback_without_a_device():
    """Without a GPU every compute entry point must fail loudly (B2_ERR_NO_DEVICE), never fall back."""
    from mitsuba_b200 import api
    if api.device_count() > 0:
        pytest.skip("a CUDA device is present")
    with pytest.raises(api.B2Error) as e:
        api.Context(0)
    assert "no CUDA device" in str(e.value) or "[2]" in str(e.value)


def test_film_develop_host_math():
    """fmtconv.cpp:979-990: rgb = spec * (w != 0 ? 1/w : w)."""
    import numpy as np
    from mitsuba_b200 import api
    film = np.zeros((2, 2, 5), np.float32)
    film[0, 0] = [2, 4, 6, 1, 2]; film[0, 1] = [1, 1, 1, 0, 0]; film[1, 0] = [3, 0, 0, 3, 3]
    rgb = api.develop(film)
    assert np.allclose(rgb[0, 0], [1, 2, 3]) and np.allclose(rgb[0, 1], 0) and np.allclose(rgb[1, 0], [1, 0, 0])


def test_product_does_not_import_the_oracle():
    """Nothing under mitsuba_b200/ may reference oracle/ (the oracle is the checker, not a backend)."""
    bad = []
    for d, _, files in os.walk(os.path.join(ROOT, "mitsuba_b200")):
        if "_obj" in d:
            continue
        for f in files:
            if f.endswith((".py", ".cpp", ".cu", ".cuh", ".h", ".inl")):
                txt = open(os.path.join(d, f), errors="ignore").read()
                if re.search(r"oracle/|oracle_api|libmtsoracle|import oracle|from oracle|\borc_", txt):
                    bad.append(os.path.join(d, f))
    assert not bad, bad


def test_wide_bvh_builder_selftest():
    """Host-side check of the 8-wide compressed tree (no device): every leaf position referenced exactly once by both trees, and a walk with
    the device's arithmetic reaches every primitive whose own box a ray hits (conservative quantisation), incl. axis-parallel rays."""
    import ctypes as C
    from mitsuba_b200 import api
    L = api.lib()
    for n, seed, rays in ((1, 1, 10), (3, 2, 10), (4, 3, 50), (17, 4, 300), (1000, 5, 400), (30000, 6, 150)):
        assert L.b2_bvh_selftest(C.c_uint32(n), C.c_uint32(seed), C.c_uint32(rays)) == 0, n


def test_mitsuba_side_plugin_propagates_library_errors_as_mitsuba_exceptions():
    """The compiled Mitsuba-side plugin (class B200PathTracer, oracle/_ref/libb200shim.so): on a machine without a CUDA device the C-ABI's
    B2_ERR_NO_DEVICE comes back through Log(EError) -> std::runtime_error, the way every Mitsuba plugin reports an error."""
    import ctypes as C
    import sys
    so = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "oracle", "_ref", "libb200shim.so")
    if not os.path.exists(so):
        pytest.skip("oracle/_ref/libb200shim.so not built (the reference tree is not on this machine)")
    from mitsuba_b200 import api
    if api.lib().b2_device_count() > 0:
        pytest.skip("a CUDA device is present: tests/test_gpu_shim.py renders through the plugin")
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import ref_pins
    lib = C.CDLL(so)
    desc, rp = next((d, r) for n, d, r in ref_pins.image_cases() if n == "cbox_box_8spp")
    h = ref_pins.reference_scene(lib, desc, rp)
    out = np.zeros((desc.camera.height, desc.camera.width, 5), np.float32)
    err = C.create_string_buffer(1024)
    lib.pathref_render_b200.restype = C.c_int
    rc = lib.pathref_render_b200(h, 0, 1, out.ctypes.data_as(C.POINTER(C.c_float)), err, 1024)
    assert rc == 1 and b"no CUDA device" in err.value


def test_bvh_build_does_not_depend_on_the_thread_count():
    """The host builder splits big nodes over threads (bounds, bins, stable partition) and hands subtrees to threads: min / max / counts
    and a stable partition are order-free, so 1 thread and many must give byte-identical trees (binary nodes, 8-wide nodes, leaf order)."""
    import ctypes as C
    from mitsuba_b200 import api
    L = api.lib()
    L.b2_bvh_thread_invariance.restype = C.c_int
    for n, ta, tb in ((300000, 1, 8), (500000, 3, 16)):
        assert L.b2_bvh_thread_invariance(C.c_uint32(n), C.c_uint32(n + 1), ta, tb) == 0, (n, ta, tb)
