"""ctypes binding of libcczero_b200.so (include/cczero_b200.h).

`get_lib()` loads the nvcc-built library and raises if it is missing — there is no CPU fallback in
the product.  `CzLib(path)` is also used by the CPU test tier to bind the emulator build of the same kernels,
which executes the same integer-kernel source under a SIMT emulator (test tier only).
"""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
CUDA_LIB_PATH = os.path.join(HERE, "libcczero_b200.so")

BOARD_STRIDE = 96
MAX_MOVES = 128
N_LABELS = 2086
MAX_NO_ACT = 16


class CzError(RuntimeError):
    pass


class CzConfig(C.Structure):
    _fields_ = [
        ("struct_bytes", C.c_int32), ("device", C.c_int32), ("n_games", C.c_int32),
        ("sims_per_move", C.c_int32), ("leaves_per_round", C.c_int32), ("virtual_loss", C.c_int32),
        ("max_nodes_per_game", C.c_int32), ("max_edges_per_game", C.c_int32), ("max_path", C.c_int32),
        ("noise_mode", C.c_int32), ("max_plies", C.c_int32), ("nn_filters", C.c_int32),
        ("nn_blocks", C.c_int32), ("nn_value_fc", C.c_int32),
        ("c_puct", C.c_double), ("noise_eps", C.c_double), ("dirichlet_alpha", C.c_double),
        ("tau_decay_rate", C.c_double), ("resign_threshold", C.c_double), ("enable_resign_rate", C.c_double),
        ("min_resign_turn", C.c_int32), ("max_game_length", C.c_int32),
        ("seed", C.c_uint64), ("rank", C.c_int32), ("arena", C.c_int32), ("nn_fp32_skip", C.c_int32), ("use_history", C.c_int32),
        ("game_quota", C.c_int32), ("playouts_lo", C.c_int32), ("playouts_hi", C.c_int32),
        ("nn_policy_channels", C.c_int32), ("nn_value_channels", C.c_int32), ("record_visits", C.c_int32),
        ("eval_mirror", C.c_int32),
    ]


class CzRootOpts(C.Structure):
    _fields_ = [
        ("struct_bytes", C.c_int32), ("reserved", C.c_int32),
        ("no_act_host", C.c_void_p), ("increase_temp_host", C.c_void_p), ("active_host", C.c_void_p),
        ("noise_dev", C.c_void_p), ("noise_stride", C.c_int64),
        ("sims_override", C.c_int32), ("raw_tasks", C.c_int32),
        ("root_hist_host", C.c_void_p), ("root_hist_given_host", C.c_void_p),
    ]


class CzRootInfo(C.Structure):
    _fields_ = [
        ("n_moves", C.c_int32), ("sum_n", C.c_int32), ("noise_used", C.c_int32), ("sims_run", C.c_int32),
        ("moves", C.c_uint16 * MAX_MOVES), ("n", C.c_int32 * MAX_MOVES),
        ("w", C.c_double * MAX_MOVES), ("p", C.c_float * MAX_MOVES),
    ]


MAX_PV = 32


class CzPvInfo(C.Structure):
    _fields_ = [("n_moves", C.c_int32), ("has_value", C.c_int32), ("value", C.c_float), ("moves", C.c_uint16 * MAX_PV)]


class CzRecordHdr(C.Structure):
    _fields_ = [("n_plies", C.c_int32), ("value_red", C.c_int32), ("game_index", C.c_int32), ("flags", C.c_int32)]


class CzTensorDesc(C.Structure):
    _fields_ = [("name", C.c_char_p), ("dev", C.c_void_p), ("numel", C.c_int64)]


class CzTrainConfig(C.Structure):
    _fields_ = [("struct_bytes", C.c_int32), ("filters", C.c_int32), ("blocks", C.c_int32), ("in_planes", C.c_int32),
                ("policy_channels", C.c_int32), ("value_channels", C.c_int32), ("value_fc", C.c_int32),
                ("max_batch", C.c_int32)]


class CzTrainHparams(C.Structure):
    _fields_ = [("struct_bytes", C.c_int32), ("lr", C.c_float), ("momentum", C.c_float), ("w_policy", C.c_float),
                ("w_value", C.c_float), ("l2", C.c_float)]


_P = C.c_void_p
_SIGS = {
    "cz_last_error": (C.c_char_p, []),
    "cz_build_is_cuda": (C.c_int, []),
    "cz_action_labels": (C.c_int, [_P, _P]),
    "cz_mirror_labels": (C.c_int, [_P]),
    "cz_env_movegen": (C.c_int, [_P, C.c_int, _P, _P, _P]),
    "cz_env_done": (C.c_int, [_P, C.c_int, C.c_int, _P, _P, _P]),
    "cz_env_step": (C.c_int, [_P, _P, C.c_int, _P, _P, _P]),
    "cz_env_encode_planes": (C.c_int, [_P, C.c_int, _P, _P]),
    "cz_env_check_catch": (C.c_int, [_P, _P, C.c_int, _P, _P, _P, _P]),
    "cz_env_keys": (C.c_int, [_P, C.c_int, _P, _P]),
    "cz_env_mirror": (C.c_int, [_P, _P, C.c_int, _P, _P]),
    "cz_sl_replay": (C.c_int, [_P, _P, _P, _P, C.c_int, C.c_int, _P, _P, _P, _P, _P]),
    "cz_play_replay": (C.c_int, [_P, _P, _P, C.c_int, _P, _P, _P, _P, _P]),
    "cz_workspace_bytes": (C.c_int, [C.POINTER(CzConfig), C.POINTER(C.c_uint64)]),
    "cz_create": (C.c_int, [C.POINTER(CzConfig), _P, C.c_uint64, _P, C.POINTER(_P)]),
    "cz_destroy": (None, [_P]),
    "cz_reset_games": (C.c_int, [_P, _P]),
    "cz_set_root": (C.c_int, [_P, C.c_int, _P]),
    "cz_set_roots": (C.c_int, [_P, _P]),
    "cz_get_roots": (C.c_int, [_P, _P]),
    "cz_get_root_stats": (C.c_int, [_P, _P, _P, _P, _P]),
    "cz_compact": (C.c_int, [_P]),
    "cz_search_begin": (C.c_int, [_P, C.POINTER(CzRootOpts)]),
    "cz_search_more": (C.c_int, [_P, C.c_int32]),
    "cz_set_noise_table": (C.c_int, [_P, _P, C.c_int64]),
    "cz_get_pv": (C.c_int, [_P, C.c_int, C.c_int32, C.POINTER(CzPvInfo)]),
    "cz_search_wave": (C.c_int, [_P, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "cz_leaf_planes": (C.c_int, [_P, _P]),
    "cz_leaf_boards": (C.c_int, [_P, _P]),
    "cz_search_apply": (C.c_int, [_P, _P, _P]),
    "cz_leaf_labels": (C.c_int, [_P, _P, _P]),
    "cz_search_apply_legal": (C.c_int, [_P, _P, _P]),
    "cz_search": (C.c_int, [_P, C.POINTER(CzRootOpts)]),
    "cz_search_run": (C.c_int, [_P]),
    "cz_get_root": (C.c_int, [_P, C.c_int, C.POINTER(CzRootInfo)]),
    "cz_get_counters": (C.c_int, [_P, _P]),
    "cz_get_search_stats": (C.c_int, [_P, _P]),
    "cz_play_move": (C.c_int, [_P, C.POINTER(C.c_int32)]),
    "cz_selfplay": (C.c_int, [_P, C.c_int32, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int64)]),
    "cz_set_game_sims": (C.c_int, [_P, _P]),
    "cz_get_active": (C.c_int, [_P, _P]),
    "cz_record_layout": (C.c_int, [_P, _P]),
    "cz_clear_records": (C.c_int, [_P]),
    "cz_drain_records": (C.c_int, [_P, _P, _P, C.c_int32, C.POINTER(C.c_int32)]),
    "cz_record_buffer": (C.c_int, [_P, C.POINTER(_P), C.POINTER(C.c_uint64), C.POINTER(C.c_int32)]),
    "cz_drain_records_visits": (C.c_int, [_P, _P, _P, _P, _P, C.c_int64, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int64)]),
    "cz_record_visits_buffer": (C.c_int, [_P, C.POINTER(_P), C.POINTER(C.c_uint64)]),
    "cz_record_visits_layout": (C.c_int, [_P, _P]),
    "cz_visit_targets": (C.c_int, [_P, _P, _P, _P, _P, C.c_int, _P, _P]),
    "cz_nn_set_weights": (C.c_int, [_P, C.POINTER(CzTensorDesc), C.c_int32]),
    "cz_nn_set_weights_net": (C.c_int, [_P, C.c_int32, C.POINTER(CzTensorDesc), C.c_int32]),
    "cz_nn_forward": (C.c_int, [_P, _P, C.c_int32, _P, _P]),
    "cz_nn_forward_boards": (C.c_int, [_P, _P, C.c_int32, _P, _P]),
    "cz_launch_count": (C.c_int, [_P, C.POINTER(C.c_uint64)]),
    "cz_nn_profile": (C.c_int, [_P, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_uint64), C.POINTER(C.c_double)]),
    "cz_noise_sample": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, _P]),
    "cz_igemm_conv3x3_dense": (C.c_int, [_P, _P, _P, _P, _P, C.c_int, C.c_int, C.c_int, _P]),
    "cz_igemm_dense": (C.c_int, [_P, _P, _P, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P]),
    "cz_nn_read_buffer": (C.c_int, [_P, C.c_int32, C.c_int32, _P, C.c_int64, C.POINTER(C.c_int64)]),
    "cz_train_workspace_bytes": (C.c_int, [C.POINTER(CzTrainConfig), C.POINTER(C.c_uint64)]),
    "cz_train_create": (C.c_int, [C.POINTER(CzTrainConfig), _P, C.c_uint64, _P, C.POINTER(_P)]),
    "cz_train_destroy": (None, [_P]),
    "cz_train_set_params": (C.c_int, [_P, C.POINTER(CzTensorDesc), C.c_int32, C.POINTER(CzTensorDesc), C.c_int32]),
    "cz_train_step": (C.c_int, [_P, _P, _P, _P, C.c_int32, C.POINTER(CzTrainHparams), _P]),
    "cz_train_read_grad": (C.c_int, [_P, C.c_char_p, _P, C.c_int64]),
    "cz_train_read_buffer": (C.c_int, [_P, C.c_int32, C.c_int32, _P, C.c_int64, C.POINTER(C.c_int64)]),
    "cz_train_set_adam": (C.c_int, [_P, C.POINTER(CzTensorDesc), C.c_int32, C.POINTER(CzTensorDesc), C.c_int32, C.c_double,
                                    C.c_double, C.c_double]),
    "cz_train_adam_iterations": (C.c_int, [_P, C.POINTER(C.c_int64)]),
    "cz_train_wgrad3x3": (C.c_int, [_P, _P, C.c_int, C.c_int, _P, _P]),
    "cz_train_dgrad3x3": (C.c_int, [_P, _P, C.c_int, C.c_int, _P, _P]),
    "cz_train_bn": (C.c_int, [_P, C.c_longlong, C.c_int, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
}
# entry points that only exist in the CUDA build (tensor cores cannot be emulated on the CPU)
CUDA_ONLY = {"cz_igemm_conv3x3_dense", "cz_igemm_dense", "cz_train_workspace_bytes", "cz_train_create",
             "cz_train_destroy", "cz_train_set_params", "cz_train_step", "cz_train_read_grad", "cz_train_read_buffer", "cz_train_wgrad3x3",
             "cz_train_dgrad3x3", "cz_train_bn", "cz_train_set_adam", "cz_train_adam_iterations"}


class CzLib:
    """Thin typed view of the shared library; every call raises CzError on a negative status."""

    def __init__(self, path):
        if not os.path.exists(path):
            raise CzError(
                f"native library missing: {path} — build it with "
                "`python chinesechess-alphazero_b200/build.py cuda` (there is no CPU fallback)")
        self.path = path
        self._dll = C.CDLL(path, mode=C.RTLD_LOCAL)
        self.missing = []
        for name, (res, args) in _SIGS.items():
            try:
                fn = getattr(self._dll, name)
            except AttributeError:
                self.missing.append(name)
                continue
            fn.restype = res
            fn.argtypes = args
        self.is_cuda = bool(self._dll.cz_build_is_cuda())

    def raw(self, name):
        return getattr(self._dll, name)

    def call(self, name, *args):
        rc = getattr(self._dll, name)(*args)
        if rc is not None and rc < 0:
            msg = self._dll.cz_last_error()
            raise CzError(f"{name} failed ({rc}): {msg.decode() if msg else ''}")
        return rc


_lib = None


def get_lib():
    """The product library (CUDA).  Builds it with nvcc if the in-tree .so is missing (a fresh clone); raises CzError when
    that is not possible.  There is no CPU fallback."""
    global _lib
    if _lib is None:
        if not os.path.exists(CUDA_LIB_PATH):
            try:
                from . import build
                build.build_cuda()
            except Exception as e:       # no nvcc, compile error ...
                raise CzError(f"native library missing and could not be built ({e}); run "
                              "`python chinesechess-alphazero_b200/build.py cuda`") from e
        _lib = CzLib(CUDA_LIB_PATH)
        if not _lib.is_cuda:
            raise CzError("libcczero_b200.so is not a CUDA build")
    return _lib
