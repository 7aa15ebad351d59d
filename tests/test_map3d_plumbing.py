"""What the three 3-D maps (TruncatedSignedDistanceMap, OccupancyMap3D, DynamicDistanceMap3D) share through the device patch store.
CPU: the status of every create() refusal through the C-ABI (LAMA_ERR_ARG before any CUDA call, LAMA_ERR_NO_DEVICE without a
device).  GPU: a map reading a file written at another resolution takes the file's resolution for world points too."""
import ctypes as C

import numpy as np
import pytest

import occ3d_oracle as T

O = T.OFFSET
LAMA_ERR_ARG, LAMA_ERR_NO_DEVICE = -1, -3


def _create(api, which, window=None, **dev):
    """lama_<which>_create with a valid resolution, patch size and map argument, the given window and device options"""
    L = api.lib()
    d = api.DeviceOptions(device=0, dir_dim=64, pool_slots=0, max_beams=2048, timing=0, stream=0)
    for k, v in dev.items():
        setattr(d, k, v)
    win = None if window is None else (C.c_int32 * 3)(*window)
    h = C.c_void_p()
    arg = {"tsdm": C.c_int(1), "om3": C.c_int(0), "dm3": C.c_double(0.5)}[which]
    rc = getattr(L, "lama_%s_create" % which)(C.c_double(0.1), C.c_uint32(32), arg, None, win, C.byref(d), C.byref(h))
    if rc == 0:
        getattr(L, "lama_%s_destroy" % which)(h)
    return rc


# ---- CPU ---------------------------------------------------------------------------------------------------------------------------
def test_dm3_create_refuses_a_pool_of_2_to_the_24_slots_as_an_argument_error(api):
    assert _create(api, "dm3", pool_slots=1 << 24) == LAMA_ERR_ARG
    assert "pool_slots" in api.lib().lama_last_error().decode()


@pytest.mark.parametrize("which", ["tsdm", "om3", "dm3"])
@pytest.mark.parametrize("window", [(0, 4, 4), (4, 0, 4), (4, 4, 0), (2049, 1, 1), (1, 2049, 1), (1, 1, 2049)])
def test_create_refuses_a_window_axis_outside_1_to_2048_patches(api, which, window):
    assert _create(api, which, window) == LAMA_ERR_ARG
    assert "window" in api.lib().lama_last_error().decode()


@pytest.mark.parametrize("which, window", [("tsdm", (2048, 2048, 2)), ("om3", (256, 256, 2)), ("dm3", (256, 256, 2))])
def test_create_refuses_a_window_of_too_many_entries(api, which, window):
    assert _create(api, which, window) == LAMA_ERR_ARG      # 2^23 entries for the TSDM (at most 2^22), 2^17 for the others (2^16)


def test_tsdm_2d_create_refuses_a_bad_window_axis(api):
    L = api.lib()
    h = C.c_void_p()
    for window in [(0, 4, 1), (2049, 4, 1)]:
        w = (C.c_int32 * 3)(*window)
        assert L.lama_tsdm_create(C.c_double(0.1), C.c_uint32(32), C.c_int(0), None, w, None, C.byref(h)) == LAMA_ERR_ARG


@pytest.mark.parametrize("which", ["tsdm", "om3", "dm3"])
def test_valid_create_without_a_device_is_no_device(api, which):
    if api.device_count() > 0:
        pytest.skip("a CUDA device is present: the create succeeds")
    assert _create(api, which, (4, 4, 2), pool_slots=(1 << 24) - 1 if which == "dm3" else 0) == LAMA_ERR_NO_DEVICE


# ---- GPU ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["frequency", "logodds"])
def test_gpu_occupancy3d_read_takes_the_file_resolution_for_world_points(gpu_api, kind, tmp_path):
    rng = np.random.default_rng(11)
    clouds = [rng.uniform(-2.0, 2.0, (1500, 3)) for _ in range(3)]
    origins = rng.uniform(-0.5, 0.5, (3, 3))
    o = T.Oracle(0.1, kind)
    o.insertPointClouds(clouds, origins)
    assert o.write(tmp_path / "o.sdm")
    g = gpu_api.OccupancyMap3D(0.05, kind)
    g.read(tmp_path / "o.sdm")
    cells = (O + rng.integers(-40, 40, (20000, 3))).astype(np.uint32)
    world = (cells.astype(np.float64) - O) * 0.1           # cell centres of the 0.1 m map
    prob, flags = o.query(cells)
    assert np.array_equal(g.getProbability(world).view(np.uint64), prob.view(np.uint64))
    assert np.array_equal(g.isOccupied(world), (flags & 2) != 0)
    assert 0 < ((flags & 2) != 0).sum() < len(cells)
