"""ctypes binding of libdne.so (include/dne.h).  PyTorch tensors are only the device-memory container:
every call passes raw ``data_ptr()`` values and the current CUDA stream handle across the C ABI.

There is no CPU fallback: if the library is missing, or there is no CUDA device, calls raise.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("DNE_LIB") or os.path.join(_HERE, "libdne.so")     # DNE_LIB: dev override (A/B builds)

DNE_MAX_LAYERS = 8
CONV, DENSE = 0, 1
ACT_NONE, ACT_RELU, ACT_TANH = 0, 1, 2
BN_NONE, BN_TF, BN_GPU = 0, 1, 2
OB_ATARI_U8, OB_VECTOR = 0, 1
EPISODE_CARTPOLE, EPISODE_ACROBOT, EPISODE_MOUNTAINCAR = 0, 1, 2


class LayerDesc(C.Structure):
    _fields_ = [("kind", C.c_int32), ("cin", C.c_int32), ("cout", C.c_int32), ("ksize", C.c_int32),
                ("stride", C.c_int32), ("hin", C.c_int32), ("hout", C.c_int32), ("pad", C.c_int32),
                ("act", C.c_int32), ("bn", C.c_int32), ("bn_off", C.c_int32), ("_pad", C.c_int32),
                ("off_w", C.c_int64), ("off_b", C.c_int64), ("off_beta", C.c_int64), ("off_gamma", C.c_int64)]


class NetDesc(C.Structure):
    _fields_ = [("n_layers", C.c_int32), ("ob_kind", C.c_int32), ("ob_dim", C.c_int32), ("n_out", C.c_int32),
                ("vbn_len", C.c_int32), ("_pad", C.c_int32), ("num_params", C.c_int64),
                ("layers", LayerDesc * DNE_MAX_LAYERS)]


MAZE_MAX_WALLS = 64
IMAGE_MAZE_MAX_ACTIONS = 32


class MazeDesc(C.Structure):
    _fields_ = [("n_walls", C.c_int32), ("collisions_stick", C.c_int32), ("goal", C.c_float * 2),
                ("walls", (C.c_float * 4) * MAZE_MAX_WALLS)]


class DneError(RuntimeError):
    pass


_lib = None

_P = C.c_void_p
_SIGS = {
    "dne_ctx_create": [C.c_int, C.POINTER(_P)],
    "dne_ctx_destroy": [_P],
    "dne_noise_bind": [_P, _P, C.c_int64],
    "dne_forward_ws_bytes": [C.POINTER(NetDesc), C.c_int, C.POINTER(C.c_size_t)],
    "dne_perturb_forward_conv": [_P, C.POINTER(NetDesc), _P, _P, _P, _P, _P, C.c_int, C.c_int, _P, _P, _P, _P, _P,
                                 C.c_size_t, _P],
    "dne_perturb_forward_mlp": [_P, C.POINTER(NetDesc), _P, _P, _P, _P, _P, C.c_int, C.c_int, _P, _P, _P, _P, _P,
                                C.c_size_t, _P],
    "dne_ob_stat_accumulate": [_P, C.c_int, _P, C.c_int, _P, _P, _P],
    "dne_cartpole_episodes": [_P, C.POINTER(NetDesc), _P, _P, _P, _P, C.c_int, _P, C.c_int, _P, _P, _P, _P],
    "dne_discrete_episodes": [_P, C.c_int, C.POINTER(NetDesc), _P, _P, _P, _P, C.c_int, _P, C.c_int, _P, _P, _P, _P],
    "dne_pendulum_net_supported": [C.POINTER(NetDesc)],
    "dne_pendulum_episodes": [_P, C.POINTER(NetDesc), _P, _P, _P, _P, C.c_int, _P, C.c_int, _P, _P, _P, _P, _P, _P, _P,
                              _P, _P, _P],
    "dne_maze_net_supported": [C.POINTER(NetDesc)],
    "dne_maze_episodes": [_P, C.POINTER(MazeDesc), C.POINTER(NetDesc), _P, _P, _P, _P, C.c_int, _P, C.c_int, _P, _P, _P,
                          _P, _P, _P, _P, _P, _P, _P],
    "dne_abi_maze_size": [C.POINTER(C.c_int)],
    "dne_pendulum_cluster_net_supported": [C.POINTER(NetDesc)],
    "dne_maze_cluster_net_supported": [C.POINTER(NetDesc)],
    "dne_pendulum_cluster_episodes": [_P, C.POINTER(NetDesc), _P, _P, _P, _P, C.c_int, _P, C.c_int, _P, _P, _P, _P, _P,
                                      _P, _P, _P, _P, C.c_int, _P],
    "dne_maze_cluster_episodes": [_P, C.POINTER(MazeDesc), C.POINTER(NetDesc), _P, _P, _P, _P, C.c_int, _P, C.c_int, _P,
                                  _P, _P, _P, _P, _P, _P, _P, _P, C.c_int, _P],
    "dne_pendulum_cluster_geometry": [C.POINTER(NetDesc), C.c_int, C.POINTER(C.c_int)],
    "dne_maze_cluster_geometry": [C.POINTER(NetDesc), C.c_int, C.POINTER(C.c_int)],
    "dne_pendulum_binned_net_supported": [C.POINTER(NetDesc), C.c_int],
    "dne_maze_binned_net_supported": [C.POINTER(NetDesc), C.c_int],
    "dne_pendulum_binned_episodes": [_P, C.POINTER(NetDesc), _P, _P, _P, _P, C.c_int, _P, C.c_int, _P, _P, _P, _P, _P,
                                     _P, _P, _P, _P, _P, C.c_int, C.c_int, _P],
    "dne_maze_binned_episodes": [_P, C.POINTER(MazeDesc), C.POINTER(NetDesc), _P, _P, _P, _P, C.c_int, _P, C.c_int, _P,
                                 _P, _P, _P, _P, _P, _P, _P, _P, _P, C.c_int, C.c_int, _P],
    "dne_image_maze_background": [C.POINTER(MazeDesc), _P, _P],
    "dne_image_maze_reset": [C.POINTER(MazeDesc), _P, _P, _P, C.c_int, _P, _P, _P],
    "dne_image_maze_step": [C.POINTER(MazeDesc), _P, _P, C.c_int, _P, _P, C.c_int, _P, _P, _P, _P, _P, _P],
    "dne_theta_prepare": [_P, C.POINTER(NetDesc), _P, C.c_int, _P, C.c_size_t, _P],
    "dne_theta_forget": [_P, _P],
    "dne_vbn_ws_bytes": [C.POINTER(NetDesc), C.c_int, C.c_int, C.POINTER(C.c_size_t)],
    "dne_vbn_reference_pass": [_P, C.POINTER(NetDesc), _P, _P, _P, _P, _P, C.c_int, _P, C.c_int, _P, _P,
                               C.c_size_t, _P],
    "dne_preprocess_atari": [_P, _P, _P, _P, C.c_int, C.c_int, _P],
    "dne_warp_atari_rgb": [_P, _P, C.c_int, _P],
    "dne_warp_atari_palette": [_P, _P, _P, _P, C.c_int, _P],
    "dne_centered_rank": [_P, C.c_int, _P, _P, _P],
    "dne_es_grad": [_P, _P, _P, C.c_int, C.c_int64, C.c_double, _P, C.c_int, _P],
    "dne_adam_step": [_P, _P, _P, _P, _P, C.c_int64, C.c_double, C.c_double, C.c_double, C.c_double, C.c_double,
                      C.c_int, _P, _P],
    "dne_sgd_step": [_P, _P, _P, _P, C.c_int64, C.c_double, C.c_double, C.c_double, _P, _P],
    "dne_ga_materialize": [_P, C.POINTER(NetDesc), _P, _P, C.c_int, C.POINTER(C.c_double), C.c_int, _P, _P],
    "dne_abi_sizes": [C.POINTER(C.c_int), C.POINTER(C.c_int)],
    "dne_set_option": [C.c_char_p, C.c_int],
    "dne_set_phase_events": [_P, _P, _P, C.c_int],
    "dne_profile_enable": [_P, C.c_int, C.c_int],
    "dne_profile_read": [_P, C.POINTER(C.c_int), C.POINTER(C.c_double)],
    "dne_ga_mutate": [_P, _P, C.c_int64, C.c_float, C.c_int64, _P, _P],
    "dne_ga_truncate": [_P, C.c_int, C.c_int, _P, _P],
    "dne_knn_ws_bytes": [C.c_int, C.c_int, C.POINTER(C.c_size_t)],
    "dne_knn_novelty_vec": [_P, C.c_int, _P, C.c_int, C.c_int, C.c_int, _P, _P, C.c_size_t, _P],
    "dne_knn_novelty": [_P, _P, C.c_int, _P, _P, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P, C.c_size_t, _P],
}
EXPORTS = sorted(list(_SIGS) + ["dne_last_error", "dne_version", "dne_launch_count"])


def lib():
    """Load libdne.so (built in-tree by ``__graft_entry__.build()`` / ``make -C csrc``).  Fails loudly."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise DneError(f"{LIB_PATH} not built: run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(there is no CPU fallback)")
        L = C.CDLL(LIB_PATH)
        for name, args in _SIGS.items():
            fn = getattr(L, name)
            fn.argtypes = args
            fn.restype = C.c_int
        L.dne_last_error.restype = C.c_char_p
        L.dne_last_error.argtypes = []
        L.dne_version.restype = C.c_int
        L.dne_version.argtypes = []
        L.dne_launch_count.restype = C.c_longlong
        L.dne_launch_count.argtypes = [C.c_int]
        a, b = C.c_int(), C.c_int()
        L.dne_abi_sizes(C.byref(a), C.byref(b))
        if (a.value, b.value) != (C.sizeof(LayerDesc), C.sizeof(NetDesc)):
            raise DneError(f"ABI mismatch: C structs {a.value}/{b.value} bytes, ctypes {C.sizeof(LayerDesc)}/{C.sizeof(NetDesc)}")
        L.dne_abi_maze_size(C.byref(a))
        if a.value != C.sizeof(MazeDesc):
            raise DneError(f"ABI mismatch: C dne_maze_desc {a.value} bytes, ctypes {C.sizeof(MazeDesc)}")
        _lib = L
    return _lib


_DEV_SIGS = {
    "dne_test_tc_gemm": [_P, _P, _P, C.c_int, C.c_int, _P],
    "dne_dev_tc_window": [_P, _P, _P, C.c_int, C.c_int, C.POINTER(C.c_int), C.c_int, C.c_int, C.c_int, C.c_int, _P],
}
_dev = None


def dev_lib():
    """libdne_dev.so: self-tests of the wgmma + TMA plumbing (csrc/dev/).  Tests and tools only; the
    product path never loads it."""
    global _dev
    if _dev is None:
        path = os.path.join(_HERE, "libdne_dev.so")
        if not os.path.exists(path):
            raise DneError(f"{path} not built (make -C csrc)")
        L = C.CDLL(path)
        for name, args in _DEV_SIGS.items():
            fn = getattr(L, name)
            fn.argtypes = args
            fn.restype = C.c_int
        _dev = L
    return _dev


def check(rc: int):
    if rc != 0:
        raise DneError(f"libdne error {rc}: {lib().dne_last_error().decode()}")


def ptr(t: Optional[torch.Tensor], dtype=None):
    """Raw device pointer of a contiguous CUDA tensor (None -> NULL)."""
    if t is None:
        return None
    if not t.is_cuda:
        raise DneError("libdne takes device pointers only: got a CPU tensor (no CPU fallback)")
    if not t.is_contiguous():
        raise DneError("tensor must be contiguous")
    if dtype is not None and t.dtype != dtype:
        raise DneError(f"expected {dtype}, got {t.dtype}")
    return C.c_void_p(t.data_ptr())


def stream_ptr():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def cluster_geometry(task: str, net_desc, cluster: int = 0) -> dict:
    """The launch geometry of ``dne_<task>_cluster_episodes`` (task 'pendulum' or 'maze') for a net on the current
    device: cluster size, threads and dynamic shared memory bytes per CTA, members resident at once."""
    g = (C.c_int * 4)()
    check(getattr(lib(), f"dne_{task}_cluster_geometry")(C.byref(net_desc), int(cluster), g))
    return {"cluster": g[0], "threads": g[1], "smem_bytes": g[2], "resident_members": g[3]}


class Context:
    """Owns a ``dne_ctx`` for one device (one host thread per context, like the C ABI says)."""

    def __init__(self, device: int = 0):
        if not torch.cuda.is_available():
            raise DneError("no CUDA device: libdne has no CPU fallback")
        self.device = device
        h = C.c_void_p()
        check(lib().dne_ctx_create(device, C.byref(h)))
        self.handle = h
        self._noise = None

    def bind_noise(self, noise: torch.Tensor, count: int):
        check(lib().dne_noise_bind(self.handle, ptr(noise, torch.float32), count))
        self._noise = noise     # keep alive

    def close(self):
        if getattr(self, "handle", None):
            lib().dne_ctx_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
