"""The acceleration-structure builder choice at the C-ABI, without a device: the new entry points are exported, b2_stats keeps every
earlier field at its offset with the build statistics appended, and the setters refuse a null handle or an unknown mode."""
import ctypes as C

from mitsuba_b200 import api

NEW = ("b2_scene_set_accel_build", "b2_context_set_accel_build", "b2_scene_get_accel")


def test_new_symbols_are_exported_and_listed():
    L = api.lib()
    for name in NEW:
        assert hasattr(L, name) and name in api.EXPORTS


def test_stats_layout_appends_the_build_fields():
    S = api.b2_stats
    u64 = ("samples", "rays", "shadow_rays", "path_length_sum", "bad_samples", "dim_overflow", "node_visits", "prim_tests",
           "iterations", "kernel_launches")
    for i, n in enumerate(u64):
        assert getattr(S, n).offset == 8 * i
    for i, n in enumerate(("ms_total", "ms_generate", "ms_extend", "ms_shade", "ms_occluded", "ms_film")):
        assert getattr(S, n).offset == 80 + 4 * i
    for i, n in enumerate(("n_triangles", "n_bvh_nodes", "n_generate", "n_extend", "n_shade", "n_occluded", "bytes_uploaded",
                           "pool_size", "unoccluded_shadow_rays", "bvh_node_bytes")):
        assert getattr(S, n).offset == 104 + 8 * i
    assert S.accel_build_ms.offset == 184 and S.accel_build_mode.offset == 188 and C.sizeof(S) == 192


def test_setters_refuse_null_handles_and_unknown_modes():
    L = api.lib()
    for mode in (0, 1, 2, -1):
        assert L.b2_scene_set_accel_build(None, C.c_int(mode)) == 1
        assert b"null scene" in L.b2_last_error(None)
        assert L.b2_context_set_accel_build(None, C.c_int(mode)) == 1
        assert b"null context" in L.b2_last_error(None)
    n = C.c_uint64()
    assert L.b2_scene_get_accel(None, C.c_int(0), None, C.byref(n)) == 1


def test_python_front_end_rejects_unknown_builders():
    import pytest
    with pytest.raises(api.B2Error, match="accel_build must be one of"):
        api._accel_mode("gpu")
    assert api._accel_mode("host") == 0 and api._accel_mode("device") == 1
