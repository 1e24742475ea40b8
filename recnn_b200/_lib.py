"""ctypes binding of the C ABI in include/recnn_b200.h.

The library is mandatory: there is no CPU or eager-PyTorch fallback behind
these calls.  ``lib()`` raises if librecnn_b200.so is missing or was built from
different sources (run ``python -m recnn_b200.build`` or
``__graft_entry__.build()``).
"""
from __future__ import annotations

import ctypes as C
import os

from . import build as _build

PH_VALUE_GRAD, PH_VALUE_OPT, PH_POLICY_LOSS, PH_POLICY_GRAD, PH_POLICY_OPT, PH_SOFT_UPDATE, PH_GATHER = \
    1, 2, 4, 8, 16, 32, 64
PH_FINISH = 128
PH_ALL = 255
ALGO_DDPG, ALGO_TD3 = 0, 1
OPT_EXTERNAL, OPT_SGD, OPT_ADAM, OPT_RANGER, OPT_RADAM = 0, 1, 2, 3, 4
METRIC_L2, METRIC_IP, METRIC_COS = 0, 1, 2
METRIC_L1, METRIC_LINF, METRIC_CANBERRA, METRIC_BRAYCURTIS, METRIC_CORR = 3, 4, 5, 6, 7
REINFORCE_BASIC, REINFORCE_CORRECTED, REINFORCE_TOPK = 0, 1, 2


class Dims(C.Structure):
    _fields_ = [("state_dim", C.c_int32), ("action_dim", C.c_int32), ("hidden", C.c_int32),
                ("reserved", C.c_int32)]


class DiscreteDims(C.Structure):
    _fields_ = [("state_dim", C.c_int32), ("hidden", C.c_int32), ("num_items", C.c_int32), ("reserved", C.c_int32)]


class VocabShard(C.Structure):
    _fields_ = [("item_offset", C.c_int32), ("num_items", C.c_int32), ("rank", C.c_int32), ("world", C.c_int32)]


class Net(C.Structure):
    _fields_ = [("params", C.c_void_p), ("grads", C.c_void_p), ("opt_m", C.c_void_p),
                ("opt_v", C.c_void_p), ("opt_t", C.c_void_p), ("opt_slow", C.c_void_p)]


class Optim(C.Structure):
    _fields_ = [("kind", C.c_int32), ("k", C.c_int32), ("lr", C.c_double), ("beta1", C.c_double),
                ("beta2", C.c_double), ("eps", C.c_double), ("weight_decay", C.c_double),
                ("momentum", C.c_double), ("alpha", C.c_double), ("n_sma_threshold", C.c_double)]


class StepArgs(C.Structure):
    _fields_ = [
        ("algo", C.c_int32), ("phases", C.c_int32), ("learn", C.c_int32), ("do_policy_step", C.c_int32),
        ("dims", Dims),
        ("n_rows", C.c_int64), ("n_rows_global", C.c_int64),
        ("state", C.c_void_p), ("next_state", C.c_void_p), ("action", C.c_void_p),
        ("table", C.c_void_p), ("n_items", C.c_int64), ("frame", C.c_int32), ("emb_dim", C.c_int32),
        ("items", C.c_void_p), ("ratings", C.c_void_p), ("reward", C.c_void_p), ("done", C.c_void_p),
        ("policy", Net), ("target_policy", Net), ("value", Net * 2), ("target_value", Net * 2),
        ("policy_optim", Optim), ("value_optim", Optim),
        ("gamma", C.c_float), ("min_value", C.c_float), ("max_value", C.c_float),
        ("noise_std", C.c_float), ("noise_clip", C.c_float), ("dropout", C.c_int32),
        ("soft_tau", C.c_double),
        ("masks", C.c_void_p * 8), ("noise", C.c_void_p), ("seed", C.c_uint64), ("rng_step", C.c_void_p),
        ("losses", C.c_void_p), ("losses_host", C.c_void_p), ("next_action_out", C.c_void_p), ("gen_action_out", C.c_void_p),
        ("next_action_in", C.c_void_p),
        ("workspace", C.c_void_p), ("workspace_bytes", C.c_int64),
        ("comm", C.c_void_p),
    ]


class DiscreteValueArgs(C.Structure):
    _fields_ = [
        ("dims", Dims), ("policy_dims", DiscreteDims),
        ("learn", C.c_int32), ("dropout", C.c_int32), ("chunk_items", C.c_int32), ("reserved", C.c_int32),
        ("n_rows", C.c_int64),
        ("state", C.c_void_p), ("next_state", C.c_void_p), ("action", C.c_void_p), ("reward", C.c_void_p),
        ("done", C.c_void_p),
        ("value", Net), ("target_value", Net), ("target_policy", C.c_void_p),
        ("value_optim", Optim),
        ("gamma", C.c_float), ("min_value", C.c_float), ("max_value", C.c_float), ("reserved2", C.c_int32),
        ("masks", C.c_void_p * 2), ("seed", C.c_uint64), ("rng_step", C.c_void_p),
        ("losses", C.c_void_p), ("losses_host", C.c_void_p),
        ("workspace", C.c_void_p), ("workspace_bytes", C.c_int64),
    ]


class BetaDims(C.Structure):
    _fields_ = [("state_dim", C.c_int32), ("num_items", C.c_int32), ("reserved", C.c_int32 * 2)]


class BetaArgs(C.Structure):
    _fields_ = [
        ("dims", BetaDims), ("n_rows", C.c_int64), ("chunk_items", C.c_int32), ("n_rows_global", C.c_int32),
        ("net", Net), ("optim", Optim),
        ("state", C.c_void_p), ("state_ld", C.c_int64), ("action", C.c_void_p), ("probs_out", C.c_void_p),
        ("loss", C.c_void_p), ("error", C.c_void_p),
        ("workspace", C.c_void_p), ("workspace_bytes", C.c_int64),
    ]


class IvfIndex(C.Structure):
    _fields_ = [
        ("n_items", C.c_int64), ("dim", C.c_int32), ("metric", C.c_int32), ("nlist", C.c_int32),
        ("reserved", C.c_int32), ("centroids", C.c_void_p), ("centroid_norms", C.c_void_p),
        ("list_offsets", C.c_void_p), ("list_ids", C.c_void_p), ("list_table", C.c_void_p), ("list_norms", C.c_void_p),
    ]


class IvfBuildArgs(C.Structure):
    _fields_ = [
        ("index", IvfIndex), ("table", C.c_void_p), ("sample_ids", C.c_void_p), ("n_sample", C.c_int64),
        ("init", C.c_void_p), ("n_iter", C.c_int32), ("reserved", C.c_int32),
        ("workspace", C.c_void_p), ("workspace_bytes", C.c_int64),
    ]


class IvfSearchArgs(C.Structure):
    _fields_ = [
        ("index", IvfIndex), ("queries", C.c_void_p), ("n_queries", C.c_int64), ("nprobe", C.c_int32),
        ("k", C.c_int32), ("set_ids", C.c_void_p), ("n_set_ids", C.c_int64), ("set_offsets", C.c_void_p),
        ("n_sets", C.c_int64), ("row_set", C.c_void_p), ("ids_out", C.c_void_p), ("dist_out", C.c_void_p),
        ("error_flag", C.c_void_p), ("workspace", C.c_void_p), ("workspace_bytes", C.c_int64),
    ]


# the fields recnn_offsetof_ivf_*_args(i) reports, in order
IVF_BUILD_PROBE_FIELDS = ["index", "table", "sample_ids", "n_sample", "init", "n_iter", "workspace", "workspace_bytes"]
IVF_SEARCH_PROBE_FIELDS = ["index", "queries", "n_queries", "nprobe", "k", "set_ids", "n_set_ids", "set_offsets",
                           "n_sets", "row_set", "ids_out", "dist_out", "error_flag", "workspace", "workspace_bytes"]


def ivf_index(n_items, dim, metric, nlist, centroids, centroid_norms, list_offsets, list_ids, list_table, list_norms):
    """an IvfIndex over device tensors (None -> NULL)"""
    return IvfIndex(n_items, dim, metric, nlist, 0, ptr(centroids), ptr(centroid_norms), ptr(list_offsets),
                    ptr(list_ids), ptr(list_table), ptr(list_norms))


class IvfPqIndex(C.Structure):
    _fields_ = [
        ("n_items", C.c_int64), ("dim", C.c_int32), ("metric", C.c_int32), ("nlist", C.c_int32), ("m", C.c_int32),
        ("centroids", C.c_void_p), ("centroid_norms", C.c_void_p), ("list_offsets", C.c_void_p),
        ("list_ids", C.c_void_p), ("codebooks", C.c_void_p), ("codes", C.c_void_p),
    ]


class IvfPqBuildArgs(C.Structure):
    _fields_ = [
        ("index", IvfPqIndex), ("table", C.c_void_p), ("sample_ids", C.c_void_p), ("n_sample", C.c_int64),
        ("init", C.c_void_p), ("pq_init", C.c_void_p), ("n_iter", C.c_int32), ("reserved", C.c_int32),
        ("workspace", C.c_void_p), ("workspace_bytes", C.c_int64),
    ]


class IvfPqEncodeArgs(C.Structure):
    _fields_ = [("index", IvfPqIndex), ("table", C.c_void_p), ("workspace", C.c_void_p),
                ("workspace_bytes", C.c_int64)]


class IvfPqSearchArgs(C.Structure):
    _fields_ = [
        ("index", IvfPqIndex), ("table", C.c_void_p), ("norms", C.c_void_p), ("queries", C.c_void_p),
        ("n_queries", C.c_int64), ("nprobe", C.c_int32), ("k", C.c_int32), ("refine", C.c_int32),
        ("reserved", C.c_int32), ("set_ids", C.c_void_p), ("n_set_ids", C.c_int64), ("set_offsets", C.c_void_p),
        ("n_sets", C.c_int64), ("row_set", C.c_void_p), ("ids_out", C.c_void_p), ("dist_out", C.c_void_p),
        ("error_flag", C.c_void_p), ("workspace", C.c_void_p), ("workspace_bytes", C.c_int64),
    ]


# the fields recnn_offsetof_ivf_pq_*_args(i) reports, in order
IVF_PQ_BUILD_PROBE_FIELDS = ["index", "table", "sample_ids", "n_sample", "init", "pq_init", "n_iter", "workspace",
                             "workspace_bytes"]
IVF_PQ_ENCODE_PROBE_FIELDS = ["index", "table", "workspace", "workspace_bytes"]
IVF_PQ_SEARCH_PROBE_FIELDS = ["index", "table", "norms", "queries", "n_queries", "nprobe", "k", "refine", "set_ids",
                              "n_set_ids", "set_offsets", "n_sets", "row_set", "ids_out", "dist_out", "error_flag",
                              "workspace", "workspace_bytes"]


def ivf_pq_index(n_items, dim, metric, nlist, m, centroids, centroid_norms, list_offsets, list_ids, codebooks, codes):
    """an IvfPqIndex over device tensors (None -> NULL)"""
    return IvfPqIndex(n_items, dim, metric, nlist, m, ptr(centroids), ptr(centroid_norms), ptr(list_offsets),
                      ptr(list_ids), ptr(codebooks), ptr(codes))


class GraphIndex(C.Structure):
    _fields_ = [
        ("n_items", C.c_int64), ("dim", C.c_int32), ("metric", C.c_int32), ("degree", C.c_int32),
        ("n_entry", C.c_int32), ("table", C.c_void_p), ("norms", C.c_void_p), ("graph", C.c_void_p),
        ("entry", C.c_void_p),
    ]


class GraphBuildArgs(C.Structure):
    _fields_ = [
        ("index", GraphIndex), ("knn", C.c_void_p), ("knn_degree", C.c_int32), ("reserved", C.c_int32),
        ("error_flag", C.c_void_p), ("workspace", C.c_void_p), ("workspace_bytes", C.c_int64),
    ]


class GraphSearchArgs(C.Structure):
    _fields_ = [
        ("index", GraphIndex), ("queries", C.c_void_p), ("n_queries", C.c_int64), ("k", C.c_int32),
        ("itopk", C.c_int32), ("search_width", C.c_int32), ("max_iterations", C.c_int32), ("set_ids", C.c_void_p),
        ("n_set_ids", C.c_int64), ("set_offsets", C.c_void_p), ("n_sets", C.c_int64), ("row_set", C.c_void_p),
        ("ids_out", C.c_void_p), ("dist_out", C.c_void_p), ("iterations_out", C.c_void_p), ("error_flag", C.c_void_p),
        ("workspace", C.c_void_p), ("workspace_bytes", C.c_int64),
    ]


# the fields recnn_offsetof_graph_*_args(i) reports, in order
GRAPH_BUILD_PROBE_FIELDS = ["index", "knn", "knn_degree", "error_flag", "workspace", "workspace_bytes"]
GRAPH_SEARCH_PROBE_FIELDS = ["index", "queries", "n_queries", "k", "itopk", "search_width", "max_iterations",
                             "set_ids", "n_set_ids", "set_offsets", "n_sets", "row_set", "ids_out", "dist_out",
                             "iterations_out", "error_flag", "workspace", "workspace_bytes"]


def graph_index(n_items, dim, metric, degree, table, norms, graph, entry):
    """a GraphIndex over device tensors (None -> NULL); n_entry is entry's length"""
    return GraphIndex(n_items, dim, metric, degree, 0 if entry is None else int(entry.numel()), ptr(table),
                      ptr(norms), ptr(graph), ptr(entry))


_BETA_PROBE_FIELDS = ["dims", "n_rows", "net", "optim", "state", "action", "probs_out", "loss", "error",
                      "workspace_bytes", "n_rows_global"]

_PROBE_FIELDS =["dims", "n_rows", "table", "policy", "policy_optim", "gamma", "soft_tau", "masks", "seed",
                 "losses", "workspace_bytes", "comm"]

# name -> (restype, argtypes); every symbol include/recnn_b200.h declares
SIGNATURES = {
    "recnn_b200_abi_version": (C.c_int, []),
    "recnn_b200_last_error": (C.c_char_p, []),
    "recnn_b200_launch_count": (C.c_int64, []),
    "recnn_sizeof_step_args": (C.c_int64, []),
    "recnn_offsetof_step_args": (C.c_int64, [C.c_int]),
    "recnn_frame_gather": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_int,
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "recnn_done_from_sizes": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_int64, C.c_void_p]),
    "recnn_window_gather_users": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p,
                                            C.c_int64, C.c_int, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.c_void_p, C.c_void_p, C.c_void_p]),
    "recnn_window_gather_ids": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p,
                                          C.c_int, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_void_p]),
    "recnn_user_states": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                     C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "recnn_actor_param_count": (C.c_int64, [C.POINTER(Dims)]),
    "recnn_critic_param_count": (C.c_int64, [C.POINTER(Dims)]),
    "recnn_net_layout": (C.c_int, [C.POINTER(Dims), C.c_int, C.POINTER(C.c_int64)]),
    "recnn_forward_scratch_floats": (C.c_int64, [C.POINTER(Dims), C.c_int64, C.c_int]),
    "recnn_actor_forward": (C.c_int, [C.POINTER(Dims), C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p,
                                      C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "recnn_critic_forward": (C.c_int, [C.POINTER(Dims), C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "recnn_linear_forward": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                       C.c_void_p, C.c_void_p]),
    "recnn_gemm_tf32x3": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_int64,
                                    C.c_int, C.c_void_p, C.c_int64, C.c_int, C.c_void_p]),
    "recnn_gemm_fp32": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_int64,
                                  C.c_int, C.c_void_p, C.c_int64, C.c_void_p]),
    "recnn_polyak_update": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_double, C.c_void_p]),
    "recnn_step_workspace_bytes": (C.c_int64, [C.POINTER(Dims), C.c_int64, C.c_int32]),
    "recnn_ddpg_step": (C.c_int, [C.POINTER(StepArgs), C.c_void_p]),
    "recnn_td3_step": (C.c_int, [C.POINTER(StepArgs), C.c_void_p]),
    "recnn_optimizer_step": (C.c_int, [C.POINTER(Optim), C.POINTER(Net), C.c_int64, C.c_void_p, C.c_void_p]),
    "recnn_item_norms": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "recnn_retrieve_workspace_bytes": (C.c_int64, [C.c_int64, C.c_int64, C.c_int32]),
    "recnn_retrieve_topk": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int64, C.c_void_p, C.c_int32,
                                      C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "recnn_retrieve_topk_sets": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int64, C.c_void_p,
                                           C.c_int32, C.c_int32, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64,
                                           C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                           C.c_void_p]),
    "recnn_retrieve_rank_workspace_bytes": (C.c_int64, [C.c_int64, C.c_int64]),
    "recnn_retrieve_rank": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int64, C.c_void_p, C.c_int32,
                                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "recnn_retrieve_rank_sets": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int64, C.c_void_p,
                                           C.c_int32, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64,
                                           C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "recnn_sizeof_ivf_index": (C.c_int64, []),
    "recnn_sizeof_ivf_build_args": (C.c_int64, []),
    "recnn_offsetof_ivf_build_args": (C.c_int64, [C.c_int]),
    "recnn_ivf_build_workspace_bytes": (C.c_int64, [C.c_int64, C.c_int32, C.c_int32, C.c_int64]),
    "recnn_ivf_build": (C.c_int, [C.POINTER(IvfBuildArgs), C.c_void_p]),
    "recnn_ivf_list_table": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p]),
    "recnn_sizeof_ivf_search_args": (C.c_int64, []),
    "recnn_offsetof_ivf_search_args": (C.c_int64, [C.c_int]),
    "recnn_ivf_search_workspace_bytes": (C.c_int64, [C.c_int64, C.c_int32, C.c_int32, C.c_int32]),
    "recnn_ivf_search": (C.c_int, [C.POINTER(IvfSearchArgs), C.c_void_p]),
    "recnn_sizeof_ivf_pq_index": (C.c_int64, []),
    "recnn_sizeof_ivf_pq_build_args": (C.c_int64, []),
    "recnn_offsetof_ivf_pq_build_args": (C.c_int64, [C.c_int]),
    "recnn_ivf_pq_build_workspace_bytes": (C.c_int64, [C.c_int64, C.c_int32, C.c_int32, C.c_int64, C.c_int32]),
    "recnn_ivf_pq_build": (C.c_int, [C.POINTER(IvfPqBuildArgs), C.c_void_p]),
    "recnn_sizeof_ivf_pq_encode_args": (C.c_int64, []),
    "recnn_offsetof_ivf_pq_encode_args": (C.c_int64, [C.c_int]),
    "recnn_ivf_pq_encode_workspace_bytes": (C.c_int64, [C.c_int64, C.c_int32]),
    "recnn_ivf_pq_encode": (C.c_int, [C.POINTER(IvfPqEncodeArgs), C.c_void_p]),
    "recnn_sizeof_ivf_pq_search_args": (C.c_int64, []),
    "recnn_offsetof_ivf_pq_search_args": (C.c_int64, [C.c_int]),
    "recnn_ivf_pq_search_workspace_bytes": (C.c_int64, [C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    "recnn_ivf_pq_search": (C.c_int, [C.POINTER(IvfPqSearchArgs), C.c_void_p]),
    "recnn_sizeof_graph_index": (C.c_int64, []),
    "recnn_sizeof_graph_build_args": (C.c_int64, []),
    "recnn_offsetof_graph_build_args": (C.c_int64, [C.c_int]),
    "recnn_graph_build_workspace_bytes": (C.c_int64, [C.c_int64, C.c_int32]),
    "recnn_graph_build": (C.c_int, [C.POINTER(GraphBuildArgs), C.c_void_p]),
    "recnn_sizeof_graph_search_args": (C.c_int64, []),
    "recnn_offsetof_graph_search_args": (C.c_int64, [C.c_int]),
    "recnn_graph_search_workspace_bytes": (C.c_int64, [C.c_int64, C.c_int32]),
    "recnn_graph_search": (C.c_int, [C.POINTER(GraphSearchArgs), C.c_void_p]),
    "recnn_slate_distances": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int64, C.c_int32, C.c_int32,
                                        C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "recnn_slate_diversify": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_void_p, C.c_int64,
                                        C.c_int32, C.c_int32, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_void_p]),
    "recnn_critic_serve_workspace_bytes": (C.c_int64, [C.POINTER(Dims), C.c_int64, C.c_int64, C.c_int64, C.c_int32,
                                                       C.c_int32]),
    "recnn_critic_topk": (C.c_int, [C.POINTER(Dims), C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64,
                                    C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64,
                                    C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                    C.c_void_p]),
    "recnn_critic_rank": (C.c_int, [C.POINTER(Dims), C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64,
                                    C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64,
                                    C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "recnn_discrete_layout": (C.c_int, [C.POINTER(DiscreteDims), C.POINTER(C.c_int64)]),
    "recnn_discrete_scratch_floats": (C.c_int64, [C.POINTER(DiscreteDims), C.c_int64, C.c_int32]),
    "recnn_discrete_forward": (C.c_int, [C.POINTER(DiscreteDims), C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p,
                                         C.c_void_p, C.c_void_p]),
    "recnn_categorical_sample": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_int64, C.c_void_p, C.c_uint64,
                                           C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "recnn_categorical_sample_at": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_int64, C.c_void_p, C.c_uint64,
                                              C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "recnn_categorical_log_prob": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p,
                                             C.c_void_p, C.c_void_p]),
    "recnn_reinforce_policy_grad": (C.c_int, [C.POINTER(DiscreteDims), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                              C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_void_p,
                                              C.c_void_p, C.c_void_p]),
    "recnn_reinforce_policy_grad_chunked": (C.c_int, [C.POINTER(DiscreteDims), C.c_void_p, C.c_void_p, C.c_void_p,
                                                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32,
                                                      C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "recnn_reinforce_scratch_floats": (C.c_int64, [C.POINTER(DiscreteDims), C.c_int64, C.c_int32]),
    "recnn_vocab_record_floats": (C.c_int64, [C.c_int64]),
    "recnn_reinforce_shard_stats": (C.c_int, [C.POINTER(DiscreteDims), C.POINTER(VocabShard), C.c_void_p, C.c_void_p,
                                              C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "recnn_reinforce_shard_grad": (C.c_int, [C.POINTER(DiscreteDims), C.POINTER(VocabShard), C.c_void_p, C.c_void_p,
                                             C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32,
                                             C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "recnn_discrete_shard_forward": (C.c_int, [C.POINTER(DiscreteDims), C.POINTER(VocabShard), C.c_void_p, C.c_void_p,
                                               C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "recnn_discrete_shard_finish": (C.c_int, [C.POINTER(DiscreteDims), C.POINTER(VocabShard), C.c_void_p, C.c_int64,
                                              C.c_void_p, C.c_void_p, C.c_void_p]),
    "recnn_discrete_shard_sample": (C.c_int, [C.POINTER(DiscreteDims), C.POINTER(VocabShard), C.c_void_p, C.c_void_p,
                                              C.c_int64, C.c_void_p, C.c_uint64, C.c_int64, C.c_void_p, C.c_void_p]),
    "recnn_discrete_shard_log_prob": (C.c_int, [C.POINTER(DiscreteDims), C.POINTER(VocabShard), C.c_void_p, C.c_int64,
                                                C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "recnn_discrete_shard_pick": (C.c_int, [C.c_int32, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.c_void_p]),
    "recnn_discrete_topk_workspace_bytes": (C.c_int64, [C.POINTER(DiscreteDims), C.c_int64, C.c_int32, C.c_int32]),
    "recnn_discrete_topk": (C.c_int, [C.POINTER(DiscreteDims), C.c_void_p, C.c_void_p, C.c_int64, C.c_int32,
                                      C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_int64, C.c_void_p]),
    "recnn_vocab_topk_record_floats": (C.c_int64, [C.c_int64, C.c_int32]),
    "recnn_discrete_shard_topk": (C.c_int, [C.POINTER(DiscreteDims), C.POINTER(VocabShard), C.c_void_p, C.c_void_p,
                                            C.c_int64, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p,
                                            C.c_void_p, C.c_int64, C.c_void_p]),
    "recnn_discrete_shard_topk_finish": (C.c_int, [C.POINTER(DiscreteDims), C.POINTER(VocabShard), C.c_void_p,
                                                   C.c_int64, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p,
                                                   C.c_void_p, C.c_void_p, C.c_void_p]),
    "recnn_discrete_topk_sets": (C.c_int, [C.POINTER(DiscreteDims), C.c_void_p, C.c_void_p, C.c_int64, C.c_int32,
                                           C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int32,
                                           C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "recnn_discrete_shard_topk_sets": (C.c_int, [C.POINTER(DiscreteDims), C.POINTER(VocabShard), C.c_void_p,
                                                 C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int64, C.c_void_p,
                                                 C.c_int64, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                                 C.c_int64, C.c_void_p]),
    "recnn_discrete_sample_topk": (C.c_int, [C.POINTER(DiscreteDims), C.c_void_p, C.c_void_p, C.c_int64, C.c_int32,
                                             C.c_void_p, C.c_int32, C.c_uint64, C.c_int64, C.c_int32, C.c_void_p,
                                             C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "recnn_discrete_sample_topk_sets": (C.c_int, [C.POINTER(DiscreteDims), C.c_void_p, C.c_void_p, C.c_int64,
                                                  C.c_int32, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p,
                                                  C.c_uint64, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                                  C.c_void_p, C.c_int64, C.c_void_p]),
    "recnn_vocab_sample_topk_record_floats": (C.c_int64, [C.c_int64, C.c_int32]),
    "recnn_discrete_shard_sample_topk": (C.c_int, [C.POINTER(DiscreteDims), C.POINTER(VocabShard), C.c_void_p,
                                                   C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int32,
                                                   C.c_uint64, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p,
                                                   C.c_int64, C.c_void_p]),
    "recnn_discrete_shard_sample_topk_sets": (C.c_int, [C.POINTER(DiscreteDims), C.POINTER(VocabShard), C.c_void_p,
                                                        C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int64,
                                                        C.c_void_p, C.c_int64, C.c_void_p, C.c_uint64, C.c_int64,
                                                        C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                                        C.c_void_p]),
    "recnn_discrete_shard_sample_topk_finish": (C.c_int, [C.POINTER(DiscreteDims), C.POINTER(VocabShard), C.c_void_p,
                                                          C.c_int64, C.c_int32, C.c_void_p, C.c_int32, C.c_uint64,
                                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "recnn_discrete_rank_workspace_bytes": (C.c_int64, [C.POINTER(DiscreteDims), C.c_int64, C.c_int32]),
    "recnn_discrete_rank": (C.c_int, [C.POINTER(DiscreteDims), C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                      C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                      C.c_void_p]),
    "recnn_discrete_rank_sets": (C.c_int, [C.POINTER(DiscreteDims), C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                           C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int32,
                                           C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "recnn_vocab_rank_record_floats": (C.c_int64, [C.c_int64]),
    "recnn_discrete_shard_rank_stats": (C.c_int, [C.POINTER(DiscreteDims), C.POINTER(VocabShard), C.c_void_p,
                                                  C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p,
                                                  C.c_void_p, C.c_int64, C.c_void_p]),
    "recnn_discrete_shard_rank": (C.c_int, [C.POINTER(DiscreteDims), C.POINTER(VocabShard), C.c_void_p, C.c_void_p,
                                            C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                            C.c_void_p]),
    "recnn_discrete_shard_rank_sets": (C.c_int, [C.POINTER(DiscreteDims), C.POINTER(VocabShard), C.c_void_p,
                                                 C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64,
                                                 C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                                 C.c_void_p, C.c_int64, C.c_void_p]),
    "recnn_discrete_shard_rank_finish": (C.c_int, [C.POINTER(DiscreteDims), C.POINTER(VocabShard), C.c_void_p,
                                                   C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p,
                                                   C.c_void_p, C.c_void_p]),
    "recnn_discrete_log_prob": (C.c_int, [C.POINTER(DiscreteDims), C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                          C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "recnn_vocab_log_prob_finish": (C.c_int, [C.POINTER(VocabShard), C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p,
                                              C.c_void_p, C.c_void_p]),
    "recnn_critic_action_term_scratch_floats":(C.c_int64, [C.POINTER(Dims), C.POINTER(DiscreteDims), C.c_int64,
                                                            C.c_int32]),
    "recnn_critic_action_term_chunked": (C.c_int, [C.POINTER(Dims), C.c_void_p, C.POINTER(DiscreteDims), C.c_void_p,
                                                   C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_void_p,
                                                   C.c_void_p, C.c_void_p]),
    "recnn_critic_forward_action_term": (C.c_int, [C.POINTER(Dims), C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "recnn_sizeof_discrete_value_args": (C.c_int64, []),
    "recnn_discrete_value_workspace_bytes": (C.c_int64, [C.POINTER(Dims), C.POINTER(DiscreteDims), C.c_int64,
                                                         C.c_int32]),
    "recnn_discrete_value_step": (C.c_int, [C.POINTER(DiscreteValueArgs), C.c_void_p]),
    "recnn_discrete_value_dp_grad_floats": (C.c_int64, [C.POINTER(Dims)]),
    "recnn_discrete_value_dp_record_floats": (C.c_int64, [C.POINTER(Dims), C.c_int64]),
    "recnn_discrete_value_dp_workspace_bytes": (C.c_int64, [C.POINTER(Dims), C.POINTER(DiscreteDims), C.c_int64,
                                                            C.c_int64, C.c_int32]),
    "recnn_discrete_value_dp_begin": (C.c_int, [C.POINTER(DiscreteValueArgs), C.c_int64, C.c_int64, C.c_int64,
                                                C.c_void_p, C.c_void_p, C.c_void_p]),
    "recnn_discrete_value_dp_end": (C.c_int, [C.POINTER(DiscreteValueArgs), C.c_int64, C.c_int64, C.c_int32,
                                              C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "recnn_discrete_value_shard_begin": (C.c_int, [C.POINTER(DiscreteValueArgs), C.POINTER(VocabShard), C.c_void_p,
                                                   C.c_void_p]),
    "recnn_discrete_value_shard_merge": (C.c_int, [C.POINTER(DiscreteValueArgs), C.POINTER(VocabShard), C.c_void_p,
                                                   C.c_void_p, C.c_void_p]),
    "recnn_discrete_value_shard_end": (C.c_int, [C.POINTER(DiscreteValueArgs), C.POINTER(VocabShard), C.c_void_p,
                                                 C.c_void_p]),
    "recnn_beta_layout": (C.c_int, [C.POINTER(BetaDims), C.POINTER(C.c_int64)]),
    "recnn_beta_workspace_bytes": (C.c_int64, [C.POINTER(BetaDims), C.c_int64, C.c_int32]),
    "recnn_sizeof_beta_args": (C.c_int64, []),
    "recnn_offsetof_beta_args": (C.c_int64, [C.c_int]),
    "recnn_beta_step": (C.c_int, [C.POINTER(BetaArgs), C.c_void_p]),
    "recnn_beta_shard_begin": (C.c_int, [C.POINTER(BetaArgs), C.POINTER(VocabShard), C.c_void_p, C.c_void_p]),
    "recnn_beta_shard_rows": (C.c_int, [C.POINTER(BetaArgs), C.POINTER(VocabShard), C.c_void_p, C.c_void_p,
                                        C.c_void_p]),
    "recnn_beta_shard_end": (C.c_int, [C.POINTER(BetaArgs), C.POINTER(VocabShard), C.c_void_p, C.c_void_p]),
    "recnn_beta_log_prob_workspace_bytes": (C.c_int64, [C.POINTER(BetaDims), C.c_int64, C.c_int32]),
    "recnn_beta_log_prob": (C.c_int, [C.POINTER(BetaDims), C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64,
                                      C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "recnn_beta_shard_log_prob_stats": (C.c_int, [C.POINTER(BetaDims), C.POINTER(VocabShard), C.c_void_p, C.c_void_p,
                                                  C.c_int64, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p,
                                                  C.c_int64, C.c_void_p]),
    "recnn_comm_create": (C.c_int, [C.c_int32, C.c_int32, C.c_int64, C.POINTER(C.c_void_p)]),
    "recnn_comm_handle_bytes": (C.c_int32, []),
    "recnn_comm_local_handle": (C.c_int, [C.c_void_p, C.c_void_p]),
    "recnn_comm_connect": (C.c_int, [C.c_void_p, C.c_void_p]),
    "recnn_comm_allreduce": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "recnn_comm_allgather": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "recnn_comm_destroy": (C.c_int, [C.c_void_p]),
}

_LIB = None


class RecnnError(RuntimeError):
    pass


def lib_path() -> str:
    return _build.LIB


def lib():
    """The loaded shared library (built on first use if a compiler is present)."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = lib_path()
    if not os.path.isfile(path):
        try:
            _build.build()
        except Exception as exc:  # no silent fallback: the CUDA library is the product
            raise RecnnError("librecnn_b200.so is missing and could not be built: %s" % exc) from exc
    handle = C.CDLL(path)
    for name, (res, args) in SIGNATURES.items():
        try:
            fn = getattr(handle, name)
        except AttributeError as exc:
            raise RecnnError("librecnn_b200.so does not export %s (stale build?)" % name) from exc
        fn.restype = res
        fn.argtypes = args
    if handle.recnn_sizeof_step_args() != C.sizeof(StepArgs):
        raise RecnnError("recnn_step_args layout mismatch: C %d bytes, ctypes %d bytes"
                         % (handle.recnn_sizeof_step_args(), C.sizeof(StepArgs)))
    if handle.recnn_sizeof_discrete_value_args() != C.sizeof(DiscreteValueArgs):
        raise RecnnError("recnn_discrete_value_args layout mismatch: C %d bytes, ctypes %d bytes"
                         % (handle.recnn_sizeof_discrete_value_args(), C.sizeof(DiscreteValueArgs)))
    for i, f in enumerate(_PROBE_FIELDS):
        if handle.recnn_offsetof_step_args(i) != getattr(StepArgs, f).offset:
            raise RecnnError("recnn_step_args.%s offset mismatch" % f)
    if handle.recnn_sizeof_beta_args() != C.sizeof(BetaArgs):
        raise RecnnError("recnn_beta_args layout mismatch: C %d bytes, ctypes %d bytes"
                         % (handle.recnn_sizeof_beta_args(), C.sizeof(BetaArgs)))
    for i, f in enumerate(_BETA_PROBE_FIELDS):
        if handle.recnn_offsetof_beta_args(i) != getattr(BetaArgs, f).offset:
            raise RecnnError("recnn_beta_args.%s offset mismatch" % f)
    _LIB = handle
    return handle


def check(status: int):
    if status != 0:
        msg = lib().recnn_b200_last_error()
        raise RecnnError("recnn_b200 call failed (%d): %s" % (status, (msg or b"").decode()))


def ptr(t):
    """Device/host pointer of a tensor (None -> NULL)."""
    return None if t is None else t.data_ptr()


def stream_ptr(device=None):
    import torch
    return torch.cuda.current_stream(device).cuda_stream
