"""References for the occupancy distance transform (pvb_occupancy_sdf, OccupancySDF, occupancy_distance_transform).

Definition: for every voxel c of an occupancy grid, its site s(c) is the voxel of the other state (occupied for a
free c, free for an occupied c) at the smallest squared distance D(c) = |c - s|^2 in cell units, ties to the smallest
flat C-order index; the table record is {val, gx, gy, gz} = sigma {r (sqrt(D) - 1/2), (c - s) / sqrt(D)} in fp32,
sigma = -1 for an occupied voxel, every operation rounded once.

- brute(occ): (D, site) by enumerating every opposite-state voxel (small grids).
- scipy_sqdist(occ): D from scipy.ndimage.distance_transform_edt, squared and rounded (exact at these sizes).
- check_sites(occ, D, site): the site is of the other state at distance D, and no other-state voxel with a smaller
  flat index lies at distance D (enumerating the lattice offsets o with |o|^2 = D).
- record(occ, D, site, r): the numpy float32 record formula."""
import numpy as np


def _coords(shape):
    return np.stack(np.unravel_index(np.arange(int(np.prod(shape))), shape), axis=1).astype(np.int64)


def brute(occ, chunk=512):
    """(D int64 [shape], site int64 [shape]); -1 where the grid has no voxel of the other state."""
    occ = np.asarray(occ, dtype=bool)
    flat = occ.reshape(-1)
    xyz = _coords(occ.shape)
    D = np.full(flat.size, -1, np.int64)
    S = np.full(flat.size, -1, np.int64)
    for state in (False, True):
        targets = np.nonzero(flat != state)[0]          # ascending flat order: argmin keeps the smallest index
        mine = np.nonzero(flat == state)[0]
        if targets.size == 0:
            continue
        for i in range(0, mine.size, chunk):
            m = mine[i:i + chunk]
            d2 = ((xyz[m, None, :] - xyz[None, targets, :]) ** 2).sum(-1)
            j = d2.argmin(axis=1)
            D[m] = d2[np.arange(m.size), j]
            S[m] = targets[j]
    return D.reshape(occ.shape), S.reshape(occ.shape)


def scipy_sqdist(occ):
    """D int64 [shape] from scipy's exact EDT of each state (both states must be present)."""
    from scipy.ndimage import distance_transform_edt
    occ = np.asarray(occ, dtype=bool)
    to_occ = distance_transform_edt(~occ)               # free voxels: distance to the nearest occupied one
    to_free = distance_transform_edt(occ)               # occupied voxels: distance to the nearest free one
    return np.rint(np.where(occ, to_free, to_occ) ** 2).astype(np.int64)


def _offsets(d):
    """The lattice offsets o with |o|^2 = d."""
    r = int(np.sqrt(d)) + 1
    a = np.arange(-r, r + 1)
    A, B = np.meshgrid(a, a, indexing="ij")
    rem = d - A * A - B * B
    ok = rem >= 0
    c = np.rint(np.sqrt(np.where(ok, rem, 0))).astype(np.int64)
    ok &= c * c == rem
    A, B, c = A[ok], B[ok], c[ok]
    return np.concatenate([np.stack([A, B, c], 1), np.stack([A, B, -c], 1)[c > 0]])


def check_sites(occ, D, site):
    """Raise AssertionError unless every site is of the other state, at distance D, and the smallest flat index among
    the other-state voxels at that distance."""
    occ = np.asarray(occ, dtype=bool)
    shape = np.array(occ.shape)
    flat = occ.reshape(-1)
    D = np.asarray(D).reshape(-1).astype(np.int64)
    site = np.asarray(site).reshape(-1).astype(np.int64)
    xyz = _coords(occ.shape)
    assert (site >= 0).all() and (site < flat.size).all()
    assert (flat[site] != flat).all(), "a site of the voxel's own state"
    sxyz = xyz[site]
    assert (((xyz - sxyz) ** 2).sum(1) == D).all(), "a site not at distance D"
    for d in np.unique(D):
        idx = np.nonzero(D == d)[0]
        c = xyz[idx]
        for o in _offsets(int(d)):
            q = c + o
            ok = ((q >= 0) & (q < shape)).all(1)
            qf = np.ravel_multi_index(q[ok].T, occ.shape)
            other = flat[qf] != flat[idx[ok]]
            bad = other & (qf < site[idx[ok]])
            assert not bad.any(), f"a smaller other-state index at D={d}"


def record(occ, D, site, r):
    """float32 [Nvox, 4]: the table record of every voxel of the grid occ [nx, ny, nz] (numpy float32 arithmetic, each
    operation rounded once); D and site of occ's shape or flat."""
    occ = np.asarray(occ, dtype=bool)
    xyz = _coords(occ.shape)
    occ = occ.reshape(-1)
    D = np.asarray(D).reshape(-1)
    site = np.asarray(site).reshape(-1).astype(np.int64)
    sigma = np.where(occ, np.float32(-1), np.float32(1)).astype(np.float32)
    out = np.zeros((occ.size, 4), np.float32)
    ok = D >= 0
    q = np.sqrt(D[ok].astype(np.float32))
    c, s = xyz[ok], xyz[site[ok]]
    out[ok, 0] = sigma[ok] * (np.float32(r) * (q - np.float32(0.5)))
    for k in range(3):
        out[ok, 1 + k] = sigma[ok] * ((c[:, k] - s[:, k]).astype(np.float32) / q)
    out[~ok, 0] = sigma[~ok] * np.float32(np.inf)
    return out


def host_build(occ, resolution):
    """(D int32, site int32, table float32 [Nvox, 4]) of pvb_occupancy_sdf's device routines compiled for the host
    (tests/hostsim/hostsim_edt.cpp)."""
    import ctypes
    import hostsim_lib as hs
    occ = np.ascontiguousarray(np.asarray(occ) != 0, dtype=np.uint8)
    dims = (ctypes.c_int * 3)(*occ.shape)
    D = np.empty(occ.shape, np.int32)
    S = np.empty(occ.shape, np.int32)
    T = np.empty((occ.size, 4), np.float32)
    hs.lib().simedt_occupancy_sdf(hs._p(occ), dims, ctypes.c_float(resolution), hs._p(D), hs._p(S), hs._p(T))
    return D, S, T
