"""ctypes binding of libpvb.so -- the C ABI declared in include/pvb.h.

There is NO CPU fallback: importing the query path without the compiled CUDA
library raises.  torch is used for device memory and streams only; every
pointer handed to the library is `tensor.data_ptr()`.
"""
import ctypes
import os
import subprocess

import numpy as np
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
LIB_PATH = os.environ.get("PVB_LIB") or os.path.join(CSRC, "libpvb.so")   # PVB_LIB: tuning builds only
SOURCES = ["pvb_kernels.cu", "bvh_build.cpp"]
HEADERS = ["pvb_device.cuh", os.path.join("..", "..", "include", "pvb.h")]

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "-shared"]

PVB_KIND_GRID, PVB_KIND_MESH, PVB_KIND_SPHERE, PVB_KIND_BOX, PVB_KIND_CYLINDER = 0, 1, 2, 3, 4
PVB_GRID_INDEX_FP32, PVB_GRID_OOB_GT, PVB_GRID_PRUNE_OK, PVB_MESH_CLOSED, PVB_GRID_TRILINEAR = 1, 2, 4, 8, 16
PVB_MESH_SIGNED, PVB_MESH_SURFACE_NORMAL, PVB_MESH_DEFAULT, PVB_MESH_WINDING = 1, 2, 3, 4


class NativeLibraryError(RuntimeError):
    pass


def needs_build():
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS]
    return any(os.path.exists(d) and os.path.getmtime(d) > t for d in deps)


def lib_missing():
    return not os.path.exists(LIB_PATH)


def build(force=False, verbose=False):
    """nvcc-compile the sm_90a library in-tree (cross-compiles without a GPU)."""
    if not force and not needs_build():
        return LIB_PATH
    nvcc = os.environ.get("PVB_NVCC", "nvcc")
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + SOURCES + ["-o", "libpvb.so"]
    res = subprocess.run(cmd, cwd=CSRC, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if res.returncode != 0:
        raise NativeLibraryError(f"nvcc failed ({' '.join(cmd)}):\n{res.stdout}")
    if verbose:
        print(res.stdout)
    return LIB_PATH


class SdfDesc(ctypes.Structure):
    """Mirror of pvb_sdf_desc (include/pvb.h); size checked against the library at load."""
    _fields_ = [
        ("kind", ctypes.c_int32), ("flags", ctypes.c_uint32),
        ("table", ctypes.c_void_p), ("dims", ctypes.c_int32 * 3), ("_pad0", ctypes.c_int32),
        ("min64", ctypes.c_double * 3), ("res64", ctypes.c_double * 3),
        ("min32", ctypes.c_float * 3), ("res32", ctypes.c_float * 3),
        ("valid_lo", ctypes.c_float * 3), ("valid_hi", ctypes.c_float * 3),
        ("bb_min", ctypes.c_float * 3), ("bb_max", ctypes.c_float * 3),
        ("prune_margin", ctypes.c_float),
        ("n_nodes", ctypes.c_int32),
        ("nodes", ctypes.c_void_p), ("tris", ctypes.c_void_p), ("face_normals", ctypes.c_void_p),
        ("n_tris", ctypes.c_int32), ("ray_far", ctypes.c_float * 3), ("ray_seed", ctypes.c_uint32),
        ("radius", ctypes.c_float), ("inv_res32", ctypes.c_float * 3), ("idx_certain", ctypes.c_float * 3),
        ("wn_nodes", ctypes.c_void_p),
    ]

    def copy(self):
        other = SdfDesc()
        ctypes.memmove(ctypes.byref(other), ctypes.byref(self), ctypes.sizeof(SdfDesc))
        return other


class FkFrame(ctypes.Structure):
    """Mirror of pvb_fk_frame (include/pvb.h)."""
    _fields_ = [("origin", ctypes.c_float * 12), ("axis", ctypes.c_float * 3), ("joint_type", ctypes.c_int32),
                ("q_index", ctypes.c_int32), ("_pad", ctypes.c_int32 * 3)]


class FkLink(ctypes.Structure):
    """Mirror of pvb_fk_link (include/pvb.h)."""
    _fields_ = [("mesh_from_link", ctypes.c_float * 12), ("frame", ctypes.c_int32), ("slot", ctypes.c_int32),
                ("_pad", ctypes.c_int32 * 2)]


FK_FIXED, FK_REVOLUTE, FK_PRISMATIC = 0, 1, 2
FK_MAX_FRAMES, FK_MAX_LINKS = 32, 16
FK_TREE_MAX_FRAMES, FK_TREE_MAX_LINKS = 64, 64


class OutTarget(ctypes.Structure):
    """Mirror of pvb_out_target (include/pvb.h)."""
    _fields_ = [("val", ctypes.c_void_p), ("grad", ctypes.c_void_p)]


MAX_TARGETS = 8
IPC_HANDLE_BYTES = 64

_lib = None

_SIGNATURES = {
    # name: (restype, argtypes)
    "pvb_last_error": (ctypes.c_char_p, []),
    "pvb_version": (ctypes.c_int, []),
    "pvb_sizeof_sdf_desc": (ctypes.c_int, []),
    "pvb_sizeof_bvh4_node": (ctypes.c_int, []),
    "pvb_timing_enable": (ctypes.c_int, [ctypes.c_int]),
    "pvb_timing_last_ms": (ctypes.c_int, [ctypes.POINTER(ctypes.c_float)]),
    "pvb_bvh_max_nodes": (ctypes.c_int64, [ctypes.c_int64]),
    "pvb_bvh_build": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64,
                                     ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p,
                                     ctypes.POINTER(ctypes.c_int64), ctypes.POINTER(ctypes.c_int32)]),
    "pvb_mesh_query": (ctypes.c_int, [ctypes.POINTER(SdfDesc), ctypes.c_void_p, ctypes.c_int64, ctypes.c_uint32,
                                      ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                      ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p]),
    "pvb_query_workspace": (ctypes.c_int64, [ctypes.c_int64]),
    "pvb_grid_lookup": (ctypes.c_int, [ctypes.POINTER(SdfDesc), ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p,
                                       ctypes.c_void_p, ctypes.c_void_p, ctypes.c_float, ctypes.c_void_p,
                                       ctypes.c_void_p]),
    "pvb_sphere_query": (ctypes.c_int, [ctypes.c_float, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p,
                                        ctypes.c_void_p, ctypes.c_void_p]),
    "pvb_composed_query": (ctypes.c_int, [ctypes.POINTER(SdfDesc), ctypes.c_int32, ctypes.c_int32, ctypes.c_void_p,
                                          ctypes.c_int32, ctypes.c_int32, ctypes.c_int32,
                                          ctypes.c_void_p, ctypes.c_int64, ctypes.c_uint32, ctypes.c_void_p,
                                          ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "pvb_composed_query_paired": (ctypes.c_int, [ctypes.POINTER(SdfDesc), ctypes.c_int32, ctypes.c_int32,
                                                 ctypes.c_void_p, ctypes.c_int32, ctypes.c_int32, ctypes.c_int32,
                                                 ctypes.c_void_p, ctypes.c_int64, ctypes.c_uint32, ctypes.c_void_p,
                                                 ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "pvb_composed_query_swept": (ctypes.c_int, [ctypes.POINTER(SdfDesc), ctypes.c_int32, ctypes.c_int32,
                                                ctypes.c_void_p, ctypes.c_int32, ctypes.c_int32, ctypes.c_int32,
                                                ctypes.c_void_p, ctypes.c_int64, ctypes.c_uint32, ctypes.c_void_p,
                                                ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "pvb_composed_query_clearance": (ctypes.c_int, [ctypes.POINTER(SdfDesc), ctypes.c_int32, ctypes.c_int32,
                                                    ctypes.c_void_p, ctypes.c_int32, ctypes.c_int32, ctypes.c_int32,
                                                    ctypes.c_void_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_uint32,
                                                    ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                                    ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "pvb_composed_query_paired_clearance": (ctypes.c_int, [ctypes.POINTER(SdfDesc), ctypes.c_int32, ctypes.c_int32,
                                                           ctypes.c_void_p, ctypes.c_int32, ctypes.c_int32,
                                                           ctypes.c_int32, ctypes.c_void_p, ctypes.c_int64,
                                                           ctypes.c_int64, ctypes.c_uint32, ctypes.c_void_p,
                                                           ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                                           ctypes.c_void_p, ctypes.c_void_p]),
    "pvb_composed_query_self_clearance": (ctypes.c_int, [ctypes.POINTER(SdfDesc), ctypes.c_int32, ctypes.c_void_p,
                                                         ctypes.c_void_p, ctypes.c_int32, ctypes.c_int32,
                                                         ctypes.c_int32, ctypes.c_void_p, ctypes.c_int64,
                                                         ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                                         ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                                         ctypes.c_void_p, ctypes.c_void_p]),
    "pvb_collision_cost_workspace": (ctypes.c_int64, [ctypes.c_int32, ctypes.c_int32, ctypes.c_int64, ctypes.c_int64]),
    "pvb_composed_query_collision_cost": (ctypes.c_int, [ctypes.POINTER(SdfDesc), ctypes.c_int32, ctypes.c_void_p,
                                                         ctypes.c_int32, ctypes.c_int32, ctypes.c_int32,
                                                         ctypes.c_void_p, ctypes.c_int64, ctypes.c_int64,
                                                         ctypes.c_float, ctypes.c_void_p, ctypes.c_int64,
                                                         ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "pvb_composed_query_paired_collision_cost": (ctypes.c_int, [ctypes.POINTER(SdfDesc), ctypes.c_int32,
                                                                ctypes.c_void_p, ctypes.c_int32, ctypes.c_int32,
                                                                ctypes.c_int32, ctypes.c_void_p, ctypes.c_int64,
                                                                ctypes.c_int64, ctypes.c_float, ctypes.c_void_p,
                                                                ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p,
                                                                ctypes.c_void_p]),
    "pvb_composed_query_self_collision_cost":(ctypes.c_int, [ctypes.POINTER(SdfDesc), ctypes.c_int32,
                                                              ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int32,
                                                              ctypes.c_int32, ctypes.c_int32, ctypes.c_void_p,
                                                              ctypes.c_int64, ctypes.c_void_p, ctypes.c_float,
                                                              ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "pvb_composed_query_scene_clearance": (ctypes.c_int, [ctypes.POINTER(SdfDesc), ctypes.c_int32, ctypes.c_void_p,
                                                          ctypes.c_void_p, ctypes.c_int32, ctypes.c_int32,
                                                          ctypes.c_int32, ctypes.c_int32, ctypes.c_void_p,
                                                          ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p,
                                                          ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                                          ctypes.c_void_p]),
    "pvb_composed_query_scene_collision_cost": (ctypes.c_int, [ctypes.POINTER(SdfDesc), ctypes.c_int32,
                                                               ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int32,
                                                               ctypes.c_int32, ctypes.c_int32, ctypes.c_int32,
                                                               ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p,
                                                               ctypes.c_float, ctypes.c_void_p, ctypes.c_void_p,
                                                               ctypes.c_void_p]),
    "pvb_composed_query_multi":(ctypes.c_int, [ctypes.POINTER(SdfDesc), ctypes.c_int32, ctypes.c_int32,
                                                ctypes.c_void_p, ctypes.c_int32, ctypes.c_int32, ctypes.c_int32,
                                                ctypes.c_void_p, ctypes.c_int64, ctypes.c_uint32, ctypes.c_void_p,
                                                ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p]),
    "pvb_composed_query_multicast": (ctypes.c_int, [ctypes.POINTER(SdfDesc), ctypes.c_int32, ctypes.c_int32,
                                                    ctypes.c_void_p, ctypes.c_int32, ctypes.c_int32, ctypes.c_int32,
                                                    ctypes.c_void_p, ctypes.c_int64, ctypes.c_uint32, ctypes.c_void_p,
                                                    ctypes.c_void_p, ctypes.c_void_p]),
    "pvb_fk_serial": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int32, ctypes.c_void_p, ctypes.c_int32,
                                     ctypes.c_void_p, ctypes.c_int32, ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p]),
    "pvb_fk_tree": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int32, ctypes.c_void_p, ctypes.c_int32,
                                   ctypes.c_void_p, ctypes.c_int32, ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p]),
    "pvb_voxel_index": (ctypes.c_int, [ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int32,
                                       ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p]),
    "pvb_voxel_scatter": (ctypes.c_int, [ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                         ctypes.c_int32, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int32, ctypes.c_void_p,
                                         ctypes.c_double, ctypes.c_void_p, ctypes.c_void_p]),
    "pvb_voxel_gather": (ctypes.c_int, [ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                        ctypes.c_int32, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int32, ctypes.c_void_p,
                                        ctypes.c_double, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "pvb_compact_workspace": (ctypes.c_int64, [ctypes.c_int64]),
    "pvb_compact_nonempty": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int32, ctypes.c_double,
                                            ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p,
                                            ctypes.c_void_p]),
    "pvb_ipc_alloc": (ctypes.c_int, [ctypes.c_int64, ctypes.POINTER(ctypes.c_void_p)]),
    "pvb_ipc_free": (ctypes.c_int, [ctypes.c_void_p]),
    "pvb_ipc_export": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_char_p]),
    "pvb_ipc_open": (ctypes.c_int, [ctypes.c_char_p, ctypes.POINTER(ctypes.c_void_p)]),
    "pvb_ipc_close": (ctypes.c_int, [ctypes.c_void_p]),
    "pvb_memcpy_async": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p]),
    "pvb_chamfer_workspace": (ctypes.c_int64, [ctypes.c_int64]),
    "pvb_chamfer": (ctypes.c_int, [ctypes.POINTER(SdfDesc), ctypes.c_void_p, ctypes.c_int32, ctypes.c_void_p,
                                   ctypes.c_int64, ctypes.c_float, ctypes.c_void_p, ctypes.c_void_p,
                                   ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p]),
    "pvb_mesh_sample": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p,
                                       ctypes.c_int64, ctypes.c_uint64, ctypes.c_void_p, ctypes.c_void_p,
                                       ctypes.c_void_p]),
    "pvb_occupancy_sdf_workspace": (ctypes.c_int64, [ctypes.c_void_p]),
    "pvb_occupancy_sdf": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_float, ctypes.c_void_p,
                                         ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                         ctypes.c_void_p]),
    "pvb_depth_points": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int32, ctypes.c_int32, ctypes.c_int32,
                                        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_float, ctypes.c_void_p,
                                        ctypes.c_void_p]),
    "pvb_depth_carve": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int32, ctypes.c_int32, ctypes.c_int32,
                                       ctypes.c_void_p, ctypes.c_void_p, ctypes.c_float, ctypes.c_float,
                                       ctypes.c_void_p, ctypes.c_float, ctypes.c_void_p, ctypes.c_void_p,
                                       ctypes.c_void_p]),
    "pvb_depth_integrate": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int32, ctypes.c_int32, ctypes.c_int32,
                                           ctypes.c_void_p, ctypes.c_void_p, ctypes.c_float, ctypes.c_float,
                                           ctypes.c_void_p, ctypes.c_float, ctypes.c_void_p, ctypes.c_void_p,
                                           ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "pvb_ray_carve": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_void_p,
                                     ctypes.c_float, ctypes.c_float, ctypes.c_void_p, ctypes.c_float, ctypes.c_void_p,
                                     ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "pvb_occupancy_apply": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                           ctypes.c_void_p]),
    "pvb_transform_points": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int32, ctypes.c_void_p, ctypes.c_int64,
                                            ctypes.c_void_p, ctypes.c_void_p]),
    "pvb_transform_points_paired": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int32, ctypes.c_void_p, ctypes.c_int64,
                                                   ctypes.c_void_p, ctypes.c_void_p]),
}

EXPORTED_SYMBOLS = tuple(_SIGNATURES)


def lib():
    """Load libpvb.so (never builds implicitly on a GPU box: the .so ships in-tree)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise NativeLibraryError(
                f"{LIB_PATH} is missing: the CUDA library has not been built. Run "
                f"`python -c 'import __graft_entry__ as g; g.build()'` (or pytorch_volumetric_b200._native.build()). "
                f"There is no CPU fallback for the SDF query path.")
        L = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        if L.pvb_sizeof_sdf_desc() != ctypes.sizeof(SdfDesc):
            raise NativeLibraryError(f"pvb_sdf_desc layout mismatch: library {L.pvb_sizeof_sdf_desc()} B, "
                                     f"binding {ctypes.sizeof(SdfDesc)} B")
        _lib = L
    return _lib


def check(rc, what=""):
    if rc != 0:
        msg = lib().pvb_last_error().decode(errors="replace")
        raise NativeLibraryError(f"libpvb {what} failed (status {rc}): {msg}")


# ------------------------------------------------------------------ helpers

def compute_device(device=None):
    """The CUDA device queries run on.  Raises when no GPU is present."""
    if not torch.cuda.is_available():
        raise NativeLibraryError("pytorch_volumetric_b200 needs a CUDA device (H100, sm_90a); "
                                 "there is no CPU fallback for the SDF query path")
    if device is None:
        return torch.device("cuda", torch.cuda.current_device())
    device = torch.device(device)
    if device.type != "cuda":
        return torch.device("cuda", torch.cuda.current_device())
    if device.index is None:
        return torch.device("cuda", torch.cuda.current_device())
    return device


def stream_ptr(device):
    return torch.cuda.current_stream(device).cuda_stream      # int; ctypes converts it for the void* parameter


def ptr(t):
    return t.data_ptr() if t is not None else None              # int -> void* (argtypes are declared)


class on_device:
    """`with torch.cuda.device(d)` only when d is not already current (the guard costs ~8 us per call)."""
    __slots__ = ("guard",)

    def __init__(self, device):
        self.guard = None if torch.cuda.current_device() == device.index else torch.cuda.device(device)

    def __enter__(self):
        if self.guard is not None:
            self.guard.__enter__()

    def __exit__(self, *exc):
        if self.guard is not None:
            self.guard.__exit__(*exc)
        return False


def as_f32_points(points, device):
    """[..., 3] tensor/ndarray -> contiguous fp32 (M,3) on `device` (H2D copy if the input is on the host)."""
    if (torch.is_tensor(points) and points.dtype == torch.float32 and points.device == device
            and points.is_contiguous() and points.shape[-1] == 3):
        return points.detach().view(-1, 3)          # the common case: nothing to convert
    if not torch.is_tensor(points):
        points = torch.as_tensor(np.asarray(points))
    p = points.detach().reshape(-1, points.shape[-1])
    if p.shape[-1] != 3:
        raise ValueError(f"expected points with last dimension 3, got {tuple(points.shape)}")
    return p.to(device=device, dtype=torch.float32, non_blocking=True).contiguous()


def query_workspace(n, device):
    """Device scratch for the spatial binning of large tree-walk batches (None for small ones)."""
    nbytes = int(lib().pvb_query_workspace(n))
    return torch.empty(nbytes, dtype=torch.uint8, device=device) if nbytes > 0 else None


def deliver(t, device, dtype=None):
    """Move a result to the caller's device/dtype.  GPU -> host goes through pinned memory from torch's caching
    host allocator (an asynchronous copy on the current stream followed by one stream sync), which is what makes
    the host-buffer path run at PCIe speed instead of pageable-copy speed."""
    if dtype is not None and t.dtype != dtype:
        t = t.to(dtype)
    if not isinstance(device, torch.device):
        device = torch.device(device)
    if t.device == device or (device.type == "cuda" and device.index is None and t.device.type == "cuda"):
        return t
    if device.type == "cpu" and t.device.type == "cuda":
        out = torch.empty(t.shape, dtype=t.dtype, pin_memory=True)
        out.copy_(t, non_blocking=True)
        torch.cuda.current_stream(t.device).synchronize()
        return out
    return t.to(device)


def timing_enable(on=True):
    """Bracket the dominant kernel of every query call with CUDA events (include/pvb.h pvb_timing_enable)."""
    check(lib().pvb_timing_enable(1 if on else 0), "pvb_timing_enable")


def timing_last_ms():
    """Device time (ms) of the most recent dominant-kernel launch on the current device (synchronises on it)."""
    ms = ctypes.c_float(0.0)
    check(lib().pvb_timing_last_ms(ctypes.byref(ms)), "pvb_timing_last_ms")
    return float(ms.value)


def bvh_build(verts32, faces32):
    """Host BVH4 build.  Returns (nodes uint8[n_nodes,128], tris float32[F,12], max_depth)."""
    L = lib()
    verts32 = np.ascontiguousarray(verts32, dtype=np.float32)
    faces32 = np.ascontiguousarray(faces32, dtype=np.int32)
    nf = len(faces32)
    cap = int(L.pvb_bvh_max_nodes(nf))
    nodes = np.zeros((cap, 128), dtype=np.uint8)
    tris = np.zeros((nf, 12), dtype=np.float32)
    n_nodes = ctypes.c_int64(0)
    depth = ctypes.c_int32(0)
    check(L.pvb_bvh_build(verts32.ctypes.data, len(verts32), faces32.ctypes.data, nf, nodes.ctypes.data, cap,
                          tris.ctypes.data, ctypes.byref(n_nodes), ctypes.byref(depth)), "pvb_bvh_build")
    return nodes[:n_nodes.value].copy(), tris, int(depth.value)


def desc_array(descs):
    """Contiguous host array of pvb_sdf_desc for the composed kernels (passed to the kernel by value)."""
    arr = (SdfDesc * len(descs))()
    for i, d in enumerate(descs):
        ctypes.memmove(ctypes.byref(arr[i]), ctypes.byref(d), ctypes.sizeof(SdfDesc))
    return arr
