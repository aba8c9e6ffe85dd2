"""ctypes binding of libkge_b200.so (include/kge_b200.h).

There is no CPU fallback: if the shared library is missing or no CUDA device is
visible, the first use raises.  `build()` compiles the library in-tree with nvcc
(sm_90a); `load()` dlopens it and declares every prototype.
"""
import ctypes as C
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.environ.get("KGE_B200_LIB") or os.path.join(_HERE, "libkge_b200.so")  # override: kernel A/B experiments
CSRC = os.path.join(_HERE, "csrc")
HEADER = os.path.join(os.path.dirname(_HERE), "include", "kge_b200.h")

KGE_OK, KGE_ERR_INVALID_ARGUMENT, KGE_ERR_CUDA, KGE_ERR_UNSUPPORTED = 0, 1, 2, 3
SCORING = {"TransE": 0, "DistMult": 1, "ComplEx": 2, "HolE": 3, "RotatE": 4}
LOSSES = {"pairwise": 0, "nll": 1, "absolute_margin": 2, "self_adversarial": 3, "multiclass_nll": 4}
REDUCTIONS = {"sum": 0, "mean": 1}
OPTIMIZERS = {"sgd": 0, "adam": 1, "adagrad": 2, "rmsprop": 3, "adadelta": 4, "adamax": 5, "nadam": 6, "ftrl": 7}
SIDES = {"s": 0, "o": 1, "p": 2}  # "p": relation prediction, candidates are relation rows
STRATEGIES = {"worst": 0, "best": 1, "middle": 2}
STEP_FUSED, STEP_FORWARD_ONLY, STEP_BACKWARD_EXT, STEP_FUSED_DEFER = 0, 1, 2, 3
RANK_MODES = {"auto": 0, "exact": 1}
INIT_KINDS = {"uniform": 0, "normal": 1, "truncated_normal": 2, "constant": 3}
METRICS = {"euclidean": 0, "manhattan": 1}
ABI_VERSION = 2


class KgeConfig(C.Structure):
    _fields_ = [("struct_size", C.c_int32), ("scoring", C.c_int32), ("k", C.c_int32), ("eta", C.c_int32),
                ("n_ent", C.c_int64), ("n_rel", C.c_int64), ("loss", C.c_int32), ("reduction", C.c_int32),
                ("margin", C.c_float), ("alpha", C.c_float), ("device", C.c_int32), ("neg_group", C.c_int32),
                ("max_rel_size", C.c_int64), ("rank_mode", C.c_int32), ("rank_pair_cap", C.c_int32)]


class KgeOptimizerConfig(C.Structure):
    _fields_ = [("struct_size", C.c_int32), ("kind", C.c_int32), ("learning_rate", C.c_float),
                ("beta_1", C.c_float), ("beta_2", C.c_float), ("epsilon", C.c_float), ("momentum", C.c_float),
                ("initial_accumulator_value", C.c_float), ("reg_p", C.c_int32), ("reg_lambda", C.c_float),
                ("reg_p2", C.c_int32), ("reg_lambda2", C.c_float), ("rho", C.c_float), ("centered", C.c_int32),
                ("l1", C.c_float), ("l2", C.c_float), ("l2_shrinkage", C.c_float), ("lr_power", C.c_float),
                ("ftrl_beta", C.c_float), ("nadam_m_t", C.c_float), ("nadam_m_t1", C.c_float), ("nadam_s_new", C.c_float),
                ("nadam_s_next", C.c_float), ("nadam_v_den", C.c_float)]


class KgeShardMap(C.Structure):
    _fields_ = [("struct_size", C.c_int32), ("world", C.c_int32), ("rows_per_shard", C.c_int64),
                ("ent", C.c_void_p * 8), ("grad_ent", C.c_void_p * 8), ("stamp_ent", C.c_void_p * 8)]


class KgeNegativeSampler(C.Structure):
    _fields_ = [("struct_size", C.c_int32), ("max_attempts", C.c_int32), ("thresholds", C.c_void_p),
                ("sub_pool_off", C.c_void_p), ("sub_pool_ids", C.c_void_p), ("obj_pool_off", C.c_void_p),
                ("obj_pool_ids", C.c_void_p), ("sub_filter_n", C.c_int64), ("sub_filter_keys", C.c_void_p),
                ("sub_filter_vals", C.c_void_p), ("obj_filter_n", C.c_int64), ("obj_filter_keys", C.c_void_p),
                ("obj_filter_vals", C.c_void_p)]


class KgeNSCaching(C.Structure):
    _fields_ = [("struct_size", C.c_int32), ("cache_size", C.c_int32), ("random_size", C.c_int32), ("pad_", C.c_int32),
                ("sub_n_keys", C.c_int64), ("sub_ids", C.c_void_p), ("sub_count", C.c_void_p),
                ("obj_n_keys", C.c_int64), ("obj_ids", C.c_void_p), ("obj_count", C.c_void_p),
                ("sub_filter_n", C.c_int64), ("sub_filter_keys", C.c_void_p), ("sub_filter_vals", C.c_void_p),
                ("obj_filter_n", C.c_int64), ("obj_filter_keys", C.c_void_p), ("obj_filter_vals", C.c_void_p)]


_P = C.c_void_p
# name -> (restype, argtypes); kept in one table so tests can check it against the header
PROTOTYPES = {
    "kge_last_error": (C.c_char_p, []),
    "kge_abi_version": (C.c_int, []),
    "kge_create": (C.c_int, [C.POINTER(KgeConfig), C.POINTER(_P)]),
    "kge_destroy": (None, [_P]),
    "kge_internal_k": (C.c_int32, [_P]),
    "kge_half_stride": (C.c_int32, [_P]),
    "kge_row_stride": (C.c_int32, [_P]),
    "kge_pack_rows": (C.c_int, [_P, _P, _P, C.c_int64, _P]),
    "kge_unpack_rows": (C.c_int, [_P, _P, _P, C.c_int64, _P]),
    "kge_init_glorot_uniform": (C.c_int, [_P, _P, C.c_int64, C.c_uint64, _P]),
    "kge_init_table": (C.c_int, [_P, _P, C.c_int64, C.c_int32, C.c_float, C.c_float, C.c_uint64, _P]),
    "kge_score_triples": (C.c_int, [_P, _P, _P, _P, C.c_int64, _P, _P]),
    "kge_generate_corruptions": (C.c_int, [_P, _P, C.c_int64, C.c_uint64, C.c_uint64, _P, _P]),
    "kge_philox4x32_10": (None, [_P, _P, _P]),
    "kge_host_corruptions": (C.c_int, [_P, C.c_int64, C.c_int32, C.c_int64, C.c_uint64, C.c_uint64, _P]),
    "kge_sample_negatives": (C.c_int, [_P, C.POINTER(KgeNegativeSampler), _P, C.c_int64, C.c_uint64, C.c_uint64, _P, _P,
                                       _P, _P]),
    "kge_nscaching_step": (C.c_int, [_P, C.POINTER(KgeNSCaching), _P, _P, _P, _P, _P, C.c_int64, C.c_uint64, C.c_uint64,
                                     _P, _P, _P, _P]),
    "kge_shared_negatives_workspace_bytes": (C.c_int64, [_P, C.c_int64, C.c_int64]),
    "kge_shared_negatives_step": (C.c_int, [_P, C.c_int64, _P, _P, _P, _P, _P, C.c_int64, C.POINTER(KgeNegativeSampler),
                                            C.c_uint64, C.c_uint64, _P, _P, C.c_int64, _P]),
    "kge_train_step": (C.c_int, [_P, C.c_int32, _P, _P, _P, _P, _P, C.c_int64, _P, _P, C.c_uint64, C.c_uint64,
                                 _P, _P, _P, _P, _P, _P]),
    "kge_train_step_sharded": (C.c_int, [_P, C.c_int32, C.POINTER(KgeShardMap), _P, _P, _P, C.c_int64, _P, _P,
                                         C.c_uint64, C.c_uint64, _P, _P, _P, _P, _P, _P]),
    "kge_rank_sharded": (C.c_int, [_P, C.POINTER(KgeShardMap), C.c_int32, C.c_int32, C.c_int32, _P, _P, C.c_int64,
                                   _P, _P, C.c_int64, _P, _P, _P, C.c_int64, _P]),
    "kge_optimizer_step": (C.c_int, [_P, C.POINTER(KgeOptimizerConfig), C.c_int64, _P, _P, _P, _P, C.c_int64,
                                     _P, _P]),
    "kge_optimizer_step_deferred": (C.c_int, [_P, C.POINTER(KgeOptimizerConfig), C.c_int64, _P, _P, _P, _P, _P,
                                              C.c_int64, _P, _P]),
    "kge_set_row_stamps": (C.c_int, [_P, _P, _P]),
    "kge_set_row_stash": (C.c_int, [_P, _P, C.c_int64]),
    "kge_set_hot_entities": (C.c_int, [_P, _P, C.c_int32]),
    "kge_train_workspace_bytes": (C.c_int64, [_P, C.c_int64]),
    "kge_set_train_workspace": (C.c_int, [_P, _P, C.c_int64, _P]),
    "kge_rows_resident": (C.c_int, [_P]),
    "kge_step_stamp": (C.c_int32, [C.c_uint64]),
    "kge_optimizer_step_lazy": (C.c_int, [_P, C.POINTER(KgeOptimizerConfig), C.c_int64, _P, _P, _P, _P, C.c_int64, _P,
                                          C.c_int32, _P, _P]),
    "kge_optimizer_step_decay": (C.c_int, [_P, C.POINTER(KgeOptimizerConfig), C.c_int64, _P, _P, _P, _P, C.c_int64, _P,
                                           C.c_int32, _P]),
    "kge_optimizer_step_sharded": (C.c_int, [_P, C.POINTER(KgeOptimizerConfig), C.c_int64, C.c_int32, C.c_int32,
                                             C.POINTER(_P), C.POINTER(_P), _P, _P, C.c_int64, C.c_int64, _P, _P]),
    "kge_optimizer_step_exchange": (C.c_int, [_P, C.POINTER(KgeOptimizerConfig), C.POINTER(KgeOptimizerConfig), C.c_int64,
                                              C.c_int32, C.c_int32, C.POINTER(_P), C.POINTER(_P), _P, _P, _P, _P, _P,
                                              C.c_int64, C.c_int64, C.POINTER(_P), C.c_uint32, C.c_int32, _P, _P]),
    "kge_set_exchange_trace": (C.c_int, [_P, _P]),
    "kge_peer_barrier": (C.c_int, [_P, C.c_int32, C.c_int32, C.POINTER(_P), C.c_int32, C.c_uint32, _P]),
    "kge_rank": (C.c_int, [_P, C.c_int32, C.c_int32, _P, _P, _P, C.c_int64, _P, C.c_int64, C.c_int64, _P, _P,
                           C.c_int64, _P, _P, _P, C.c_int64, _P]),
    "kge_rank_finalize": (C.c_int, [_P, _P, C.c_int64, C.c_int32, _P, _P]),
    "kge_corruption_scores": (C.c_int, [_P, C.c_int32, _P, _P, _P, C.c_int64, _P, C.c_int64, C.c_int64, _P, _P,
                                        C.c_int64, _P]),
    "kge_rank_filter_probe": (C.c_int, [_P, C.c_int32, _P, _P, _P, C.c_int64, _P, C.c_int64, C.c_int64, _P, _P, _P,
                                        C.c_int64, _P]),
    "kge_rank_workspace_bytes": (C.c_int64, [_P, C.c_int64, C.c_int64]),
    "kge_topk": (C.c_int, [_P, C.c_int32, _P, _P, _P, C.c_int64, _P, C.c_int64, C.c_int64, _P, _P, C.c_int64, C.c_int32,
                           _P, _P, _P, C.c_int64, _P]),
    "kge_topk_workspace_bytes": (C.c_int64, [_P, C.c_int64, C.c_int64, C.c_int32]),
    "kge_select_topk": (C.c_int, [_P, _P, C.c_int64, C.c_int64, C.c_int32, _P, _P, _P, C.c_int64, _P]),
    "kge_select_topk_workspace_bytes": (C.c_int64, [_P, C.c_int64, C.c_int64, C.c_int32]),
    "kge_knn": (C.c_int, [_P, C.c_int32, _P, C.c_int64, C.c_int32, _P, C.c_int64, _P, C.c_int64, C.c_int64, _P, _P,
                          C.c_int64, C.c_int32, C.c_int32, _P, _P, _P, C.c_int64, _P]),
    "kge_knn_workspace_bytes": (C.c_int64, [_P, C.c_int64, C.c_int64, C.c_int32, C.c_int32]),
    "kge_radius_neighbors": (C.c_int, [_P, C.c_int32, _P, C.c_int64, C.c_int32, _P, C.c_int64, _P, C.c_int64, C.c_int64,
                                       C.c_float, _P, _P, _P, C.c_int64, _P]),
    "kge_radius_workspace_bytes": (C.c_int64, [_P, C.c_int64, C.c_int64, C.c_int32]),
    "kge_radius_union": (C.c_int, [_P, C.c_int32, _P, C.c_int64, C.c_int32, _P, C.c_int64, _P, C.c_int64, C.c_int64,
                                   C.c_float, _P, _P, C.c_int64, _P]),
    "kge_radius_min_key": (C.c_int, [_P, C.c_int32, _P, C.c_int64, C.c_int32, _P, C.c_int64, _P, C.c_int64, C.c_int64,
                                     C.c_float, _P, _P, _P, C.c_int64, _P]),
    "kge_forest_flatten": (C.c_int, [_P, _P, C.c_int64, _P]),
    "kge_graph_counts": (C.c_int, [_P, _P, _P, C.c_int64, _P, _P, _P, _P, C.c_int64, _P]),
    "kge_graph_workspace_bytes": (C.c_int64, [C.c_int64]),
    "kge_one_vs_all_workspace_bytes": (C.c_int64, [_P, C.c_int64]),
    "kge_one_vs_all_step": (C.c_int, [_P, C.c_int32, C.c_int32, _P, _P, _P, _P, _P, C.c_int64, C.c_uint64, _P, _P,
                                      C.c_int64, _P]),
    "kge_one_vs_all_relation_workspace_bytes": (C.c_int64, [_P, C.c_int64]),
    "kge_one_vs_all_relation_step": (C.c_int, [_P, C.c_float, C.c_int32, _P, _P, _P, _P, _P, C.c_int64, C.c_uint64, _P,
                                               _P, C.c_int64, _P]),
    "kge_k_vs_all_workspace_bytes": (C.c_int64, [_P, C.c_int64]),
    "kge_k_vs_all_step": (C.c_int, [_P, C.c_int32, C.c_int32, C.c_float, _P, _P, _P, _P, _P, C.c_int64, _P, _P, C.c_uint64,
                                    _P, _P, C.c_int64, _P]),
    "kge_set_embedding_dropout": (C.c_int, [_P, C.c_float, C.c_float, C.c_uint64]),
    "kge_n3_workspace_bytes": (C.c_int64, [_P]),
    "kge_n3_step": (C.c_int, [_P, C.c_float, C.c_float, _P, _P, _P, _P, _P, C.c_int64, C.c_uint64, _P, _P, C.c_int64,
                              _P]),
    "kge_dura_step": (C.c_int, [_P, C.c_float, C.c_float, _P, _P, _P, _P, _P, C.c_int64, C.c_uint64, _P, _P]),
}
ONE_VS_ALL_SIDES = {"s": 1, "o": 2, "s,o": 3}  # kge_one_vs_all_side flags of fit(one_vs_all=...)

_lib = None


def build(verbose=False):
    """Compile libkge_b200.so in-tree for sm_90a (nvcc cross-compiles without a GPU)."""
    cmd = ["make", "-C", CSRC, "-j8"]
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if verbose or out.returncode != 0:
        print(out.stdout)
    if out.returncode != 0:
        raise RuntimeError("building libkge_b200.so failed (see output above)")
    return SO_PATH


def load():
    """dlopen the library and declare prototypes.  Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(SO_PATH):
        raise RuntimeError(
            "ampligraph_b200: %s not found. Build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "or `make -C ampligraph_b200/csrc`. There is no CPU fallback for the CUDA path." % SO_PATH)
    lib = C.CDLL(SO_PATH)
    for name, (res, args) in PROTOTYPES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is missing
        fn.restype = res
        fn.argtypes = args
    if lib.kge_abi_version() != ABI_VERSION:
        raise RuntimeError("libkge_b200.so ABI version %d, binding expects %d" % (lib.kge_abi_version(), ABI_VERSION))
    _lib = lib
    return lib


def check(rc):
    """Translate a kge_status into the exception type the reference would raise."""
    if rc == KGE_OK:
        return
    msg = load().kge_last_error().decode("utf-8", "replace")
    if rc == KGE_ERR_INVALID_ARGUMENT:
        raise ValueError(msg)
    if rc == KGE_ERR_UNSUPPORTED:
        raise NotImplementedError(msg)
    raise RuntimeError(msg)


def host_corruptions(triples, eta, n_ent, seed=0, step=0):
    """CPU replay of the corruption stream of (seed, step): int32 [eta*B, 3], row j*B+i = j-th corruption of
    positive i -- bit-identical to what the fused kernel draws on the device (kge_host_corruptions)."""
    import numpy as np
    t = np.ascontiguousarray(triples, dtype=np.int32).reshape(-1, 3)
    out = np.empty((t.shape[0] * int(eta), 3), dtype=np.int32)
    check(load().kge_host_corruptions(t.ctypes.data_as(_P), t.shape[0], int(eta), int(n_ent), int(seed), int(step),
                                      out.ctypes.data_as(_P)))
    return out

