"""CPU tier of the occupancy distance transform (pvb_occupancy_sdf, OccupancySDF, occupancy_distance_transform).

1. The host build of the device routines (tests/hostsim/hostsim_edt.cpp) against brute force and scipy on random
   grids from 0.1 % to 90 % occupancy, planted ties, single-voxel grids and 1024-long lines whose breakpoint
   cross-products reach the int64 range; sites pass the lattice check.
2. Table records bit for bit against the numpy float32 formula.
3. The Python ValueErrors and the C entry point's refusals, without a GPU."""
import ctypes
import math

import numpy as np
import pytest
import torch

import edt_ref
from hostsim_lib import PVB_ERR_INVALID


def _random(shape, p, seed):
    g = np.random.default_rng(seed)
    occ = g.random(shape) < p
    i = int(g.integers(occ.size))
    occ.reshape(-1)[i] = True                              # both states present at every density
    occ.reshape(-1)[(i + 1 + int(g.integers(occ.size - 1))) % occ.size] = False
    return occ


def _check_brute(occ, resolution=0.01):
    D, S = edt_ref.brute(occ)
    d, s, t = edt_ref.host_build(occ, resolution)
    assert np.array_equal(d, D) and np.array_equal(s, S)
    assert np.array_equal(t.view(np.uint32), edt_ref.record(occ, D, S, resolution).view(np.uint32))


# ---------------------------------------------------------------- 1. the transform
@pytest.mark.parametrize("p", [0.001, 0.01, 0.05, 0.3, 0.5, 0.7, 0.9])
@pytest.mark.parametrize("shape", [(7, 9, 11), (3, 5, 70), (13, 33, 4), (40, 2, 3)])
def test_random_grids_against_brute_force(shape, p):
    _check_brute(_random(shape, p, seed=hash((shape, p)) % 2 ** 32))


@pytest.mark.parametrize("p", [0.001, 0.02, 0.3, 0.9])
def test_larger_grids_against_scipy(p):
    occ = _random((37, 45, 66), p, seed=int(p * 1000))
    d, s, _ = edt_ref.host_build(occ, 0.01)
    assert np.array_equal(d, edt_ref.scipy_sqdist(occ))
    edt_ref.check_sites(occ, d, s)


def test_planted_ties():
    """Equidistant sites in every axis order and along diagonals: the smallest flat index wins."""
    shape = (11, 11, 11)
    c = np.array([5, 5, 5])
    groups = [[(3, 0, 0), (-3, 0, 0)], [(0, 3, 0), (0, -3, 0)], [(0, 0, 3), (0, 0, -3)],
              [(3, 0, 0), (0, 3, 0), (0, 0, 3)], [(0, 0, -3), (0, -3, 0), (-3, 0, 0)],
              [(0, 0, 5), (0, 3, 4), (3, 4, 0), (4, 0, -3), (-5, 0, 0)], [(1, 1, 0), (0, -1, 1), (-1, 0, -1)],
              [(2, 2, 1), (3, 0, 0), (-1, 2, -2)]]
    for offs in groups:
        for perm in ([0, 1, 2], [2, 1, 0], [1, 2, 0]):
            occ = np.zeros(shape, bool)
            for o in offs:
                occ[tuple(c + np.asarray(o)[perm])] = True
            _check_brute(occ)
            inv = ~occ                                  # the same ties between the free voxels
            _check_brute(inv)


@pytest.mark.parametrize("shape", [(2, 2, 2), (5, 6, 7), (1024, 2, 2), (2, 2, 1024)])
def test_single_voxel_of_one_state(shape):
    for corner in [(0, 0, 0), tuple(n - 1 for n in shape)]:
        occ = np.zeros(shape, bool)
        occ[corner] = True
        _check_brute(occ)
        _check_brute(~occ)


@pytest.mark.parametrize("shape", [(1024, 2, 2), (2, 1024, 2), (2, 2, 1024)])
def test_long_lines_at_the_breakpoint_extremes(shape):
    """Sites at both ends of a 1024-long axis (breakpoint cross-products near 2^31) and sparse random sites."""
    ax = int(np.argmax(shape))
    cases = []
    for pos in ([0, 1023], [0, 1, 1022, 1023], [1023], [0], [511, 512], [3, 700, 1020]):
        occ = np.zeros(shape, bool)
        idx = [slice(None)] * 3
        idx[ax] = pos
        occ[tuple(idx)] = True
        cases.append(occ)
        off = occ.copy()
        sub = [0, 0, 0]
        sub[(ax + 1) % 3] = 1
        for p in pos:                                   # the sites of one sub-line only: f values 0 and 1 mix
            sub[ax] = p
            off[tuple(sub)] = False
        cases.append(off)
    g = np.random.default_rng(7)
    cases.append(g.random(shape) < 0.003)
    cases.append(g.random(shape) < 0.997)
    for occ in cases:
        if occ.any() and not occ.all():
            _check_brute(occ, 0.02)


# ---------------------------------------------------------------- 2. records
@pytest.mark.parametrize("resolution", [0.01, 0.02, 0.0137, 1.0, 3.3e-5])
def test_records_bit_for_bit(resolution):
    occ = _random((20, 31, 45), 0.1, seed=3)
    d, s, t = edt_ref.host_build(occ, resolution)
    want = edt_ref.record(occ, d, s, resolution)
    assert np.array_equal(t.view(np.uint32), want.view(np.uint32))
    # the zero level lies on the faces between the states: face neighbours hold +r/2 and -r/2
    r2 = np.float32(resolution) * np.float32(0.5)
    val = t[:, 0].reshape(occ.shape)
    face = occ[:, :, 1:] != occ[:, :, :-1]
    pair = np.stack([val[:, :, 1:][face], val[:, :, :-1][face]])
    assert (np.abs(pair) == r2).all() and (pair.sum(0) == 0).all()


def test_one_state_grids_have_no_field():
    for occ in (np.zeros((4, 5, 6), bool), np.ones((4, 5, 6), bool)):
        d, s, t = edt_ref.host_build(occ, 0.01)
        assert (d == -1).all() and (s == -1).all()
        sign = -1 if occ.all() else 1
        assert (t[:, 0] == sign * np.inf).all() and (t[:, 1:] == 0).all()


# ---------------------------------------------------------------- 3. refusals
def test_python_value_errors_before_device_work():
    import pytorch_volumetric_b200 as pv
    rng = [(0.0, 0.09), (0.0, 0.09), (0.0, 0.09)]
    good = torch.zeros(10, 10, 10, dtype=torch.bool)
    good[3, 4, 5] = True
    grid = pv.VoxelGrid(0.01, rng, dtype=torch.bool)
    bad_calls = [
        lambda: pv.OccupancySDF(good, 0.01, rng, interpolation="cubic"),
        lambda: pv.OccupancySDF(grid, resolution=0.01),
        lambda: pv.OccupancySDF(grid, range_per_dim=rng),
        lambda: pv.OccupancySDF(good),
        lambda: pv.OccupancySDF(good, 0.01),
        lambda: pv.OccupancySDF(good, float("nan"), rng),
        lambda: pv.OccupancySDF(good, -0.01, rng),
        lambda: pv.OccupancySDF(good, 0.01, [(0.0, 0.1)] * 3),            # an 11^3 lattice
        lambda: pv.OccupancySDF(good.float(), 0.01, rng),
        lambda: pv.OccupancySDF(torch.zeros(10, 10, 10, dtype=torch.bool), 0.01, rng),
        lambda: pv.OccupancySDF(torch.ones(10, 10, 10, dtype=torch.uint8), 0.01, rng),
        lambda: pv.OccupancySDF(grid),                                    # nothing occupied
        lambda: pv.OccupancySDF(torch.zeros(10, 10, 1, dtype=torch.bool), 0.01, [(0, 0.09), (0, 0.09), (0, 0)]),
        lambda: pv.occupancy_distance_transform(torch.zeros(4, 4, 4, dtype=torch.bool)),
        lambda: pv.occupancy_distance_transform(np.ones((4, 4, 4), bool)),
        lambda: pv.occupancy_distance_transform(np.zeros((4, 4), bool)),
        lambda: pv.occupancy_distance_transform(np.zeros((4, 4, 1025), bool)),
        lambda: pv.occupancy_distance_transform(np.zeros((4, 4, 4), np.float32)),
    ]
    for i, call in enumerate(bad_calls):
        with pytest.raises(ValueError):
            call()


def test_abi_refuses_invalid_transforms(built_lib):
    L = built_lib
    fake = ctypes.c_void_p(1 << 12)            # never dereferenced: every call below fails its argument checks
    dims = (ctypes.c_int32 * 3)(10, 20, 30)
    need = L.pvb_occupancy_sdf_workspace(dims)
    assert need == 48 * 10 * 20 * 30
    for bad in [(1, 20, 30), (10, 1025, 30), (10, 20, 0), (-5, 20, 30), (2, 2, 1 << 30)]:
        assert L.pvb_occupancy_sdf_workspace((ctypes.c_int32 * 3)(*bad)) == -1
    assert L.pvb_occupancy_sdf_workspace(None) == -1
    assert L.pvb_occupancy_sdf_workspace((ctypes.c_int32 * 3)(2, 1024, 1024)) == 48 * 2 * 1024 * 1024

    def call(occ=fake, dims=dims, r=0.01, ws=fake, ws_bytes=need, d=fake, s=fake, t=fake):
        return L.pvb_occupancy_sdf(occ, dims, r, ws, ws_bytes, d, s, t, None)

    cases = [dict(dims=None), dict(dims=(ctypes.c_int32 * 3)(10, 20, 1)),
             dict(dims=(ctypes.c_int32 * 3)(1025, 20, 30)), dict(r=0.0), dict(r=-0.01), dict(r=math.nan),
             dict(r=math.inf), dict(r=1e39), dict(ws=None), dict(ws_bytes=need - 1), dict(ws=ctypes.c_void_p((1 << 12) + 4)),
             dict(occ=None), dict(d=None, s=None, t=None), dict(t=ctypes.c_void_p((1 << 12) + 8))]
    for kw in cases:
        assert call(**kw) == PVB_ERR_INVALID, kw
        assert L.pvb_last_error().startswith(b"pvb_occupancy_sdf"), kw
    assert b"2..1024" in (call(dims=(ctypes.c_int32 * 3)(10, 20, 1)), L.pvb_last_error())[1]
    assert b"finite and positive" in (call(r=math.nan), L.pvb_last_error())[1]
    assert b"workspace" in (call(ws_bytes=need - 1), L.pvb_last_error())[1]
    assert b"all null" in (call(d=None, s=None, t=None), L.pvb_last_error())[1]
