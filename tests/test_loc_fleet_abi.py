"""The C-ABI of Loc2DFleet without a GPU: every entry point refuses a null handle with a status and a message, a fleet cannot be
created without a device (no CPU fallback), and the Python wrapper packs lama_locf_update's arguments as include/lama_b200.h declares."""
import ctypes as C

import numpy as np
import pytest


def test_null_handles_are_refused(api):
    L = api.lib()
    null = C.c_void_p(None)
    xyr = (C.c_double * 3)()
    i = C.c_int(0)
    one = (C.c_int * 1)(0)
    opts = api.Loc2DFleet.Options()
    calls = [
        (L.lama_locf_create, (None, C.c_int(2), C.byref(null))),
        (L.lama_locf_create, (C.byref(opts), C.c_int(2), None)),
        (L.lama_locf_create, (C.byref(opts), C.c_int(0), C.byref(C.c_void_p()))),
        (L.lama_locf_distance_map, (null, C.byref(C.c_void_p()))),
        (L.lama_locf_occupancy_set, (null, None, C.c_int(0), C.c_int(1))),
        (L.lama_locf_occupancy_read, (null, b"x.sdm")),
        (L.lama_locf_set_pose, (null, C.c_int(0), xyr)),
        (L.lama_locf_set_seed, (null, C.c_int(0), C.c_uint32(1))),
        (L.lama_locf_trigger_global_localization, (null, C.c_int(0))),
        (L.lama_locf_global_localization_active, (null, C.c_int(0), C.byref(i))),
        (L.lama_locf_update, (null, C.c_int(1), one, xyr, one, None, None, xyr, None, one)),
        (L.lama_locf_get, (null, None, None, None, None)),
    ]
    for fn, args in calls:
        fn.restype = C.c_int
        L.lama_last_error().decode()
        assert fn(*args) == -1, fn.__name__
        assert len(L.lama_last_error()) > 0, fn.__name__
    assert L.lama_locf_destroy(null) == 0   # as lama_loc_destroy: destroying nothing is not an error


def test_no_cpu_fallback_without_a_device(api):
    if api.device_count() > 0:
        pytest.skip("a CUDA device is present")
    with pytest.raises(api.LamaError) as e:
        api.Loc2DFleet(api.Loc2DFleet.Options(), 4)
    assert e.value.code == -3


def test_update_arguments_follow_the_header_layout(api):
    from iris_lama_b200.api import _fleet_update_args
    s0, s1 = np.arange(6.0).reshape(2, 3), np.arange(100.0, 109.0).reshape(3, 3)
    rb, pts, n, org, qt, od, fo = _fleet_update_args([4, 1], [s0, s1], [(1, 2, 3), (4, 5, 6)], force=[True, False],
                                                     origins=[(0.1, 0.2, 0.3), (0.4, 0.5, 0.6)], quats=[(0, 0, 0, 1), (0, 0, 1, 0)])
    assert rb.dtype == np.int32 and rb.tolist() == [4, 1]
    assert n.dtype == np.int32 and n.tolist() == [2, 3]
    assert pts.dtype == np.float64 and pts.flags.c_contiguous and pts.shape == (5, 3)
    assert (pts.reshape(-1) == np.concatenate([s0.reshape(-1), s1.reshape(-1)])).all()   # the scans back to back, xyz
    assert od.shape == (2, 3) and od.flags.c_contiguous and od.reshape(-1).tolist() == [1, 2, 3, 4, 5, 6]
    assert fo.dtype == np.int32 and fo.tolist() == [1, 0]
    assert org.shape == (2, 3) and org.reshape(-1)[3] == 0.4
    assert qt.shape == (2, 4) and qt.reshape(-1).tolist() == [0, 0, 0, 1, 0, 0, 1, 0]
    none = _fleet_update_args([0], [s0], [(0, 0, 0)])
    assert none[3] is None and none[4] is None and none[6] is None   # NULL origins, quats and force
    with pytest.raises(ValueError):
        _fleet_update_args([0, 1], [s0], [(0, 0, 0), (0, 0, 0)])
