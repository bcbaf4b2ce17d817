"""ctypes binding of libplslam_b200.so (include/plslam_b200.h).

There is NO CPU fallback: if the shared library is missing it is built with nvcc; if that is
impossible, or no CUDA device is present when a context is created, an exception is raised.
"""
import ctypes as C
import logging
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("PLS_LIB_PATH", os.path.join(_HERE, "libplslam_b200.so"))  # override: development A/B builds

PLS_OK, PLS_E_INVALID, PLS_E_CUDA, PLS_E_SINGULAR, PLS_W_TINY_RESIDUAL, PLS_E_STATE, PLS_E_COMM = range(7)
SCHEMES = {"default": 0, "least_square": 1, "huber": 2, "exp": 3, "neighborhood": 4, "geman_mcclure": 5,
           "square_geman_mcclure": 6, "cauchy": 7}
MAP_KDTREE, MAP_PROJECTIVE = 0, 1
INPUT_NDARRAY, INPUT_TENSOR, INPUT_VERTEX_MAP, INPUT_NDARRAY_F64, INPUT_TENSOR_F64 = 0, 1, 2, 3, 4
PTR_DEVICE, PTR_HOST = 0x100, 0x200  # residency hints OR-ed into a layout
MAX_SEQUENCES = 64  # PLS_MAX_SEQUENCES: contexts one pls_process_frames call advances
EVAL_STATS = 32  # PLS_EVAL_STATS: doubles per pose of pls_kdmap_evaluate_poses


class PlsConfig(C.Structure):
    _fields_ = [("height", C.c_int32), ("width", C.c_int32), ("up_fov_deg", C.c_float), ("down_fov_deg", C.c_float),
                ("local_map_type", C.c_int32), ("local_map_size", C.c_int32), ("num_neighbors_normals", C.c_int32),
                ("normals_kernel_size", C.c_int32), ("scheme", C.c_int32), ("sigma", C.c_float),
                ("gn_max_iters", C.c_int32), ("gn_norm_stop", C.c_float), ("max_num_alignments", C.c_int32),
                ("threshold_delta_pose", C.c_float), ("threshold_trans", C.c_float), ("threshold_rot", C.c_float),
                ("device", C.c_int32), ("stream", C.c_void_p)]


_P, _I, _L, _D, _F = C.c_void_p, C.c_int, C.c_int64, C.c_double, C.c_float
_SIGNATURES = {
    "pls_config_default": [C.POINTER(PlsConfig)],
    "pls_create": [C.POINTER(PlsConfig), C.POINTER(_P)],
    "pls_destroy": [_P],
    "pls_synchronize": [_P],
    "pls_wait_stream": [_P, _P],
    "pls_voxel_hash": [_P, _P, _I, _L, _D, _P, _P],
    "pls_voxel_hash_xyz": [_P, _P, _I, _L, _D, _D, _D, _P, _P],
    "pls_grid_sample": [_P, _P, _I, _L, _D, _P, _P, C.POINTER(_L)],
    "pls_grid_sample_staged": [_P, _P, _I, _L, _D, C.POINTER(_P), C.POINTER(_P), C.POINTER(_P), C.POINTER(_L)],
    "pls_host_fingerprint": [_P, _L, C.POINTER(C.c_uint64)],
    "pls_pinned_alloc": [_L, C.POINTER(_P)],
    "pls_pinned_free": [_P],
    "pls_project_pixels": [_P, _P, _L, _I, _I, _F, _F, _P],
    "pls_build_projection_map": [_P, _P, _P, _I, _L, _I, _I, _I, _F, _F, _P],
    "pls_build_projection_map_filled": [_P, _P, _P, _I, _L, _I, _I, _I, _F, _F, _F, _P],
    "pls_normal_map": [_P, _P, _I, _I, _I, _I, _P],
    "pls_compute_neighbors": [_P, _P, _P, _P, _I, _I, _I, _I, _P, _P],
    "pls_build_pose_matrix": [_P, _P, _I, _P],
    "pls_from_pose_matrix": [_P, _P, _I, _P],
    "pls_align_p2plane": [_P, _P, _P, _P, _L, _I, _I, _D, _I, _D, _P, _P, _P, _P],
    "pls_distort": [_P, _P, _I, _P, _I, _L, _P, _I, _P],
    "pls_voxel_statistics": [_P, _P, _I, _L, _D, _P, _P, _P, _P, _P, _P, C.POINTER(_L)],
    "pls_align_p2point": [_P, _P, _P, _L, _I, _I, _D, _I, _D, _P, _P, _P, _P],
    "pls_align_p2plane_batch": [_P, _P, _P, _P, _L, _L, _I, _I, _D, _I, _D, _P, _P, _P, _P, _P],
    "pls_align_p2point_batch": [_P, _P, _P, _L, _L, _I, _I, _D, _I, _D, _P, _P, _P, _P, _P],
    "pls_weighted_procrustes": [_P, _P, _P, _P, _L, _I, _P],
    "pls_p2plane_loss": [_P, _P, _P, _P, _P, _P, _I, _I, _I, _F, _F, _I, _F, _P, _P, _P, _P],
    "pls_kitti_correct_scan": [_P, _P, _L, _I, _P],
    "pls_ingest_scan": [_P, _P, _L, _I, _I, _I, _I, _F, _F, _P, _P],
    "pls_relative_poses": [_P, _P, _L, _I, _P],
    "pls_absolute_poses": [_P, _P, _L, _I, _P],
    "pls_map_init": [_P],
    "pls_kdmap_update_points": [_P, _P, _P, _L],
    "pls_kdmap_update_vertex_map": [_P, _P, _P, _I, _I],
    "pls_kdmap_size": [_P, C.POINTER(_L)],
    "pls_kdmap_stats": [_P, _P],
    "pls_kdmap_points": [_P, _P],
    "pls_kdmap_nn_search": [_P, _P, _L, _P, _P, _P],
    "pls_kdmap_last_correspondences": [_P, _L, _P, _P, _P, _P, _P],
    "pls_kdmap_knn": [_P, _P, _L, _I, _P, _P, _P],
    "pls_kdmap_set_points": [_P, _P, _I, _L],
    "pls_kdmap_frames": [_P, _P, C.POINTER(_I)],
    "pls_kdmap_pose_search": [_P, _P, _L, _P, _I, _D, _I, _I, _I, _P, _P, _P, _P, C.POINTER(_I)],
    "pls_kdmap_pose_search_pyramid": [_P, _P, _L, _P, _I, _D, _I, _I, _I, _P, _P, _P, C.POINTER(_I)],
    "pls_kdmap_pose_search_scans": [_P, _P, _P, _I, _P, _P, _D, _P, _P, _I, _P, _P, _P, _P, _P],
    "pls_projmap_last_frame": [_P, _P],
    "pls_projmap_update": [_P, _P, _P],
    "pls_projmap_num_frames": [_P, C.POINTER(_I)],
    "pls_projmap_model": [_P, _P, _P],
    "pls_projmap_nn_search": [_P, _P, _L, _P, _P, _P, C.POINTER(_L)],
    "pls_odometry_init": [_P],
    "pls_register_frame": [_P, _P, _L, _P, _P, _P, _P, C.POINTER(_I)],
    "pls_register_hypotheses": [_P, _P, _L, _P, _I, _P, _P, _P, _P, _P],
    "pls_register_scans": [_P, _P, _P, _I, _P, _P, _I, _P, _P, _P, _P, _P],
    "pls_register_scans_gated": [_P, _P, _P, _I, _P, _P, _I, _D, _P, _P, _P, _P, _P, _P],
    "pls_register_scans_degeneracy": [_P, _P, _P, _I, _P, _P, _I, _D, _D, _P, _P, _P, _P, _P, _P, _P, _P],
    "pls_kdmap_evaluate_poses": [_P, _P, _P, _I, _P, _P, _I, _D, _P],
    "pls_process_frame": [_P, _P, _I, _L, _P, _P, _P, C.POINTER(_I), _P],
    "pls_process_frame_grid_sample": [_P, _P, _L, _D, _I, _P, _P, _P, C.POINTER(_I), _P],
    "pls_process_frames": [_P, _I, _P, _P, _P, _D, _P, _P, _P, _P, _P, _P],
    "pls_last_icp_sums": [_P, _P, C.POINTER(_I)],
    "pls_comm_init": [_P, _I, _I, _P, C.c_char_p],
    "pls_comm_unique_id": [C.c_char_p, _P],
    "pls_comm_p2p_handle": [_P, _I, _P],
    "pls_comm_p2p_init": [_P, _I, _I, _P],
    "pls_comm_destroy": [_P],
    "pls_set_shard_min": [_L],
    "pls_last_sharded": [_P, C.POINTER(_I)],
    "pls_launch_count": [C.POINTER(_L)],
    "pls_profile_enable": [_P, _I, _I],
    "pls_profile_read": [_P, _I, C.POINTER(_D), C.POINTER(_L), C.POINTER(_D), _I],
}

_lib = None


def load():
    """Loads (building first if needed) the shared library.  Raises if it cannot be had."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        from . import build as _build
        _build.build()
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} is missing and could not be built: the CUDA extension is required")
    lib = C.CDLL(LIB_PATH)
    for name, args in _SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the header and the library disagree
        fn.argtypes = args
        fn.restype = C.c_int
    lib.pls_last_error.argtypes = [_P]
    lib.pls_last_error.restype = C.c_char_p
    lib.pls_version.argtypes = []
    lib.pls_version.restype = C.c_char_p
    _lib = lib
    return lib


def exported_symbols():
    """Every entry point include/plslam_b200.h declares (used by the CPU-side ABI test)."""
    return sorted(list(_SIGNATURES) + ["pls_last_error", "pls_version"])


# CUDA devices whose tensors were addressed since the last library call: the producer kernels of such a tensor sit on
# PyTorch's current stream, the library runs on its own -- Context.call orders the two (pls_wait_stream) before
# launching.  Empty (one truth test per call) whenever only host memory is passed.
_cuda_inputs = set()


def ptr(x):
    """Raw address of a numpy array / torch tensor (host or CUDA) / None."""
    if x is None:
        return None
    if type(x) is np.ndarray or isinstance(x, np.ndarray):
        assert x.flags.c_contiguous, "arrays passed to the C ABI must be C-contiguous"
        return x.__array_interface__["data"][0]  # same address as x.ctypes.data without building a ctypes object
    if hasattr(x, "data_ptr"):
        assert x.is_contiguous(), "tensors passed to the C ABI must be contiguous"
        if x.is_cuda:
            _cuda_inputs.add(x.device.index or 0)
        return x.data_ptr()
    raise TypeError(f"cannot take the address of {type(x)}")


def host_view(address: int, shape, dtype) -> np.ndarray:
    """A numpy view (no copy) of library-owned host memory, e.g. the pinned staging of pls_grid_sample_staged."""
    count = 1
    for extent in shape:
        count *= int(extent)
    buf = (C.c_char * (count * np.dtype(dtype).itemsize)).from_address(address)
    return np.frombuffer(buf, dtype=dtype, count=count).reshape(shape)


class PinnedPool:
    """Page-locked, device-mapped byte buffers that become the arrays a filter hands out: the kernel writes the result
    over PCIe straight into the memory the caller receives (no staging copy, no page faults on fresh pages).  Every
    array handed out is a view of its buffer, so the buffer's reference count says when nothing refers to it any more
    (pool entry + getrefcount's own argument = 2) and it can take the next frame.  A caller that keeps every frame's
    arrays simply exhausts the pool (`limit` buffers) and gets ordinary pageable copies from then on."""
    limit = 12
    buffers: list = []

    @classmethod
    def take(cls, num_bytes: int):
        """A free buffer of at least num_bytes (uint8 array over pinned memory), or None when the pool is exhausted."""
        import sys
        pool = cls.buffers
        for i in range(len(pool)):          # by index: a loop variable would itself hold a reference
            if sys.getrefcount(pool[i]) == 2 and pool[i].nbytes >= num_bytes:
                return pool[i]
        if len(pool) >= cls.limit:
            small = [i for i in range(len(pool)) if sys.getrefcount(pool[i]) == 2 and pool[i].nbytes < num_bytes]
            if not small:
                return None
            del pool[small[0]]              # its finalizer returns the pinned memory
        lib, p = load(), _P()
        if lib.pls_pinned_alloc(num_bytes, C.byref(p)) != PLS_OK:
            return None
        buf = np.frombuffer((C.c_char * num_bytes).from_address(p.value), dtype=np.uint8)
        import weakref
        weakref.finalize(buf, lib.pls_pinned_free, p.value)
        cls.buffers.append(buf)
        return buf


def host_fingerprint(address: int, num_bytes: int) -> int:
    out = C.c_uint64(0)
    load().pls_host_fingerprint(address, num_bytes, C.byref(out))
    return out.value


class Handoff:
    """The last grid-sample result a filter handed out as a host array, with its device-resident twin.  The odometry
    recognises the array by identity (address + size + content fingerprint; the record keeps the array alive, so the
    address cannot be recycled) and passes the device copy to the library: the samples never travel back up."""
    array = None        # the numpy array given to the caller (strong reference)
    address = 0
    rows = 0
    is_f64 = False
    dev_ptr = 0
    device = -1
    fingerprint = 0

    @classmethod
    def publish(cls, array, dev_ptr, device, is_f64):
        cls.array, cls.address, cls.rows = array, array.__array_interface__["data"][0], array.shape[0]
        cls.dev_ptr, cls.device, cls.is_f64 = dev_ptr, device, is_f64
        cls.fingerprint = host_fingerprint(cls.address, array.nbytes)

    @classmethod
    def clear(cls):
        cls.array, cls.address, cls.rows, cls.dev_ptr, cls.device = None, 0, 0, 0, -1

    @classmethod
    def match(cls, address, rows, is_f64, device):
        """The device pointer to use instead of `address`, or 0."""
        if address != cls.address or rows != cls.rows or is_f64 != cls.is_f64 or device != cls.device or not cls.dev_ptr:
            return 0
        if host_fingerprint(address, cls.array.nbytes) != cls.fingerprint:
            return 0  # the caller wrote into the array: its host content is the truth
        return cls.dev_ptr


def check(ctx_handle, status):
    """Maps status codes onto the reference's error behaviour (SURVEY.md section 8b 'Errors')."""
    if status == PLS_OK:
        return status
    msg = load().pls_last_error(ctx_handle).decode() if ctx_handle else "plslam_b200 error"
    if status == PLS_W_TINY_RESIDUAL:
        logging.warning("The residual norm is lower than threshold 1e-7. "
                        "This would lead to invalid jacobian. We prefer Stopping ICP")
        return status
    if status == PLS_E_SINGULAR:
        logging.error("Invalid Jacobian in Gauss Newton minimization, the hessian is not invertible")
        raise RuntimeError("Invalid Jacobian in Gauss Newton minimization")
    if status == PLS_E_INVALID:
        raise AssertionError(msg)
    raise RuntimeError(f"plslam_b200 status {status}: {msg}")


class Context:
    """Owns one pls_context (one CUDA device, one stream, one local map + odometry state)."""

    def __init__(self, **kwargs):
        lib = load()
        cfg = PlsConfig()
        lib.pls_config_default(C.byref(cfg))
        for k, v in kwargs.items():
            if not hasattr(cfg, k):
                raise AssertionError(f"unknown pls_config field {k}")
            setattr(cfg, k, v)
        self.cfg = cfg
        self.handle = _P()
        st = lib.pls_create(C.byref(cfg), C.byref(self.handle))
        if st == PLS_E_INVALID and not 3 <= cfg.num_neighbors_normals <= 255:
            raise AssertionError(f"num_neighbors_normals must be in [3, 255], got {cfg.num_neighbors_normals}")
        if st != PLS_OK:
            raise RuntimeError(f"pls_create failed with status {st}: a CUDA device and the sm_90a library are "
                               f"required (there is no CPU fallback)")
        self.lib = lib

    def launch_count(self) -> int:
        n = C.c_int64(0)
        self.lib.pls_launch_count(C.byref(n))
        return n.value

    def profile(self, which: int, reset: bool = True):
        """(device ms, launches, algorithmic bytes) accumulated in profile slot `which`."""
        ms, n, b = C.c_double(0), C.c_int64(0), C.c_double(0)
        self.call("pls_profile_read", which, C.byref(ms), C.byref(n), C.byref(b), int(reset))
        return ms.value, n.value, b.value

    def call(self, name, *args):
        if _cuda_inputs:
            self._order_after_torch()
        return check(self.handle, getattr(self.lib, name)(self.handle, *args))

    def check(self, status):
        """Maps a status this context's last call returned onto the reference's error behaviour (see check())."""
        return check(self.handle, status)

    def process_frames(self, *args):
        """pls_process_frames(*args); its first argument is the array of context handles, this context's among them.
        Returns the status code unchecked: errors are per sequence."""
        return self.lib.pls_process_frames(*args)

    def _order_after_torch(self):
        """CUDA tensors were addressed for this call: whatever PyTorch still has in flight on its current stream
        (a .to(float32), a slice copy, a network forward pass) must finish before the library's stream reads them."""
        import torch
        devices = list(_cuda_inputs)
        _cuda_inputs.clear()
        for d in devices:
            if d == int(self.cfg.device):
                check(self.handle, self.lib.pls_wait_stream(self.handle, torch.cuda.current_stream(d).cuda_stream))
            else:
                torch.cuda.current_stream(d).synchronize()

    def close(self):
        if getattr(self, "handle", None):
            if Handoff.device == int(self.cfg.device):
                Handoff.clear()  # the device twin may live in this context
            self.lib.pls_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
