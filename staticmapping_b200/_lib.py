"""ctypes loader for libsm_b200.so (the C ABI declared in include/sm_b200.h).

There is NO CPU fallback: if the shared library is missing, or no CUDA device is visible
when a matcher is created, this raises.  (The library itself loads on a CPU-only box so
that the symbol table can be checked there.)"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# SM_B200_LIB: A/B builds for profiles/ (same ABI); the product library is libsm_b200.so
LIB_PATH = os.environ.get("SM_B200_LIB") or os.path.join(_HERE, "libsm_b200.so")


class AlignInfo(C.Structure):
    _fields_ = [("iterations", C.c_int32), ("status", C.c_int32), ("solve_path", C.c_int32),
                ("reserved", C.c_int32), ("kept", C.c_int64), ("limit", C.c_double),
                ("ms_upload", C.c_float), ("ms_prologue", C.c_float),
                ("ms_iterations", C.c_float), ("kernel_launches", C.c_int32),
                ("ms_knn", C.c_float), ("ms_accum", C.c_float), ("ms_finish", C.c_float),
                ("profiled_iterations", C.c_int32), ("evaluations", C.c_int32),
                ("trans_probability", C.c_double), ("mean_neighbors", C.c_double),
                ("aux", C.c_double * 4)]


class Pair(C.Structure):
    _fields_ = [("source", C.c_void_p), ("n_source", C.c_int64), ("target", C.c_void_p),
                ("target_normals", C.c_void_p), ("n_target", C.c_int64), ("guess", C.c_void_p),
                ("on_device", C.c_int32), ("reserved", C.c_int32)]


_lib = None

_DP = C.POINTER(C.c_double)
_IP = C.POINTER(C.c_int32)
_VP = C.c_void_p

# name -> (restype, argtypes); this table must list every symbol of include/sm_b200.h
SIGNATURES = {
    "sm_create": (C.c_int, [C.c_int, C.c_int, C.POINTER(_VP)]),
    "sm_destroy": (C.c_int, [_VP]),
    "sm_set_option": (C.c_int, [_VP, C.c_char_p, C.c_char_p]),
    "sm_print_options": (C.c_int, [_VP, C.c_char_p, C.c_int64]),
    "sm_set_inner_compensation": (C.c_int, [_VP, C.c_int32]),
    "sm_set_ndt_search_method": (C.c_int, [_VP, C.c_int32]),
    "sm_set_icp_error_minimizer": (C.c_int, [_VP, C.c_int32]),
    "sm_set_pm_surface_normals": (C.c_int, [_VP, C.c_int32]),
    "sm_set_pm_reading_sampler": (C.c_int, [_VP, C.c_int32]),
    "sm_get_pm_rand_position": (C.c_int, [_VP, _VP]),
    "sm_set_pm_rand_position": (C.c_int, [_VP, C.c_int64]),
    "sm_get_type": (C.c_int, [_VP]),
    "sm_set_input_source": (C.c_int, [_VP, _VP, C.c_int64]),
    "sm_set_input_target": (C.c_int, [_VP, _VP, _VP, C.c_int64]),
    "sm_set_input_source_f32": (C.c_int, [_VP, _VP, C.c_int64, C.c_int64]),
    "sm_set_input_target_f32": (C.c_int, [_VP, _VP, C.c_int64, C.c_int64]),
    "sm_set_input_source_f32_device": (C.c_int, [_VP, _VP, C.c_int64, C.c_int64]),
    "sm_set_input_target_f32_device": (C.c_int, [_VP, _VP, C.c_int64, C.c_int64]),
    "sm_set_input_source_device": (C.c_int, [_VP, _VP, C.c_int64]),
    "sm_set_input_target_device": (C.c_int, [_VP, _VP, _VP, C.c_int64]),
    "sm_align": (C.c_int, [_VP, _DP, _DP]),
    "sm_align_async": (C.c_int, [_VP, _DP]),
    "sm_align_wait": (C.c_int, [_VP, _DP]),
    "sm_align_batch": (C.c_int, [_VP, C.c_int32, _VP, _VP, _VP]),
    "sm_align_pairs": (C.c_int, [_VP, C.c_int32, _VP, C.c_int32, _VP, _VP, _VP]),
    "sm_get_fitness_score": (C.c_double, [_VP]),
    "sm_get_align_info": (C.c_int, [_VP, C.POINTER(AlignInfo)]),
    "sm_set_stream": (C.c_int, [_VP, _VP]),
    "sm_last_error": (C.c_char_p, [_VP]),
    "sm_knn1": (C.c_int, [C.c_int, _VP, C.c_int64, _VP, C.c_int64, C.c_double, C.c_int, _VP, _VP]),
    "sm_knn": (C.c_int, [C.c_int, _VP, C.c_int64, _VP, C.c_int64, C.c_int32, C.c_double, C.c_double, C.c_uint32,
                         C.c_int, _VP, _VP]),
    "sm_knn_device": (C.c_int, [C.c_int, _VP, C.c_int64, _VP, C.c_int64, C.c_int32, C.c_double, C.c_double,
                                C.c_uint32, C.c_int, _VP, _VP, _VP]),
    "sm_calculate_normals": (C.c_int, [C.c_int, _VP, C.c_int64, _VP, _VP, C.POINTER(C.c_int64)]),
    "sm_calculate_normals_ordered": (C.c_int, [C.c_int, _VP, C.c_int64, C.c_int32, _VP, _VP, C.POINTER(C.c_int64)]),
    "sm_motion_compensation": (C.c_int, [C.c_int, _VP, C.c_int64, C.c_int64, _DP, _VP]),
    "sm_motion_compensation_device": (C.c_int, [C.c_int, _VP, C.c_int64, C.c_int64, _DP, _VP, _VP]),
    "sm_voxel_grid_filter": (C.c_int, [C.c_int, _VP, C.c_int64, C.c_int64, C.c_float, _VP, C.POINTER(C.c_int64)]),
    "sm_voxel_grid_filter_ordered": (C.c_int, [C.c_int, _VP, C.c_int64, C.c_int64, C.c_float, C.c_int32, _VP,
                                               C.POINTER(C.c_int64)]),
    "sm_m2dp_descriptor_length": (C.c_int64, [C.c_double, C.c_double, C.c_int32, C.c_int32, C.c_int32]),
    "sm_m2dp": (C.c_int, [C.c_int, _VP, C.c_int64, C.c_int64, C.c_double, C.c_double, C.c_int32, C.c_int32, C.c_int32,
                          _VP, C.c_int64, _VP]),
    "sm_m2dp_match": (C.c_double, [_VP, _VP, C.c_int64]),
    "sm_filter_chain_create": (C.c_int, [C.c_int, C.POINTER(_VP)]),
    "sm_filter_chain_destroy": (C.c_int, [_VP]),
    "sm_filter_chain_add": (C.c_int, [_VP, C.c_char_p]),
    "sm_filter_chain_set_param": (C.c_int, [_VP, C.c_int, C.c_char_p, C.c_int, C.c_char_p]),
    "sm_filter_chain_validate": (C.c_int, [_VP, C.c_int]),
    "sm_filter_chain_set_option": (C.c_int, [_VP, C.c_char_p, C.c_char_p]),
    "sm_filter_chain_set_random_sampler": (C.c_int, [_VP, C.c_int, C.c_int32, C.c_uint32]),
    "sm_filter_chain_set_voxel_order": (C.c_int, [_VP, C.c_int, C.c_int32]),
    "sm_filter_chain_run": (C.c_int, [_VP, _VP, C.c_int64, C.c_int64, _VP, C.POINTER(C.c_int64), _VP]),
    "sm_filter_chain_run_device": (C.c_int, [_VP, _VP, C.c_int64, C.c_int64, _VP, C.POINTER(C.c_int64), _VP, _VP]),
    "sm_filter_chain_depth_cluster": (C.c_int, [_VP, C.c_int, _VP, C.c_int64, C.c_int64, _VP, _VP, _VP,
                                                C.POINTER(C.c_int64), _VP]),
    "sm_filter_chain_last_error": (C.c_char_p, [_VP]),
    "sm_statistic_removal_create": (C.c_int, [C.c_int, C.POINTER(_VP)]),
    "sm_statistic_removal_destroy": (C.c_int, [_VP]),
    "sm_statistic_removal_set_param": (C.c_int, [_VP, C.c_char_p, C.c_int, C.c_char_p]),
    "sm_statistic_removal_run": (C.c_int, [_VP, _VP, C.c_int64, C.c_int64, _VP, C.POINTER(C.c_int64), _VP]),
    "sm_statistic_removal_run_device": (C.c_int, [_VP, _VP, C.c_int64, C.c_int64, _VP, C.POINTER(C.c_int64), _VP,
                                                  _VP]),
    "sm_statistic_removal_stats": (C.c_int, [_VP, _DP]),
    "sm_statistic_removal_last_error": (C.c_char_p, [_VP]),
    "sm_ground_removal_create": (C.c_int, [C.c_int, C.POINTER(_VP)]),
    "sm_ground_removal_destroy": (C.c_int, [_VP]),
    "sm_ground_removal_set_param": (C.c_int, [_VP, C.c_char_p, C.c_int, C.c_char_p]),
    "sm_ground_removal_run": (C.c_int, [_VP, _VP, C.c_int64, C.c_int64, _VP, C.POINTER(C.c_int64), _VP]),
    "sm_ground_removal_run_device": (C.c_int, [_VP, _VP, C.c_int64, C.c_int64, _VP, C.POINTER(C.c_int64), _VP, _VP]),
    "sm_ground_removal_indices": (C.c_int, [_VP, _VP, C.POINTER(C.c_int64), _VP, C.POINTER(C.c_int64)]),
    "sm_ground_removal_last_error": (C.c_char_p, [_VP]),
    "sm_plane_sampler_create": (C.c_int, [C.c_int, C.POINTER(_VP)]),
    "sm_plane_sampler_destroy": (C.c_int, [_VP]),
    "sm_plane_sampler_set_sampling_rate": (C.c_int, [_VP, C.c_float]),
    "sm_plane_sampler_set_leaf_size": (C.c_int, [_VP, C.c_float]),
    "sm_plane_sampler_set_min_point_num_in_voxel": (C.c_int, [_VP, C.c_uint64]),
    "sm_plane_sampler_run": (C.c_int, [_VP, _VP, C.c_int64, C.c_int64, _VP, C.POINTER(C.c_int64), _VP]),
    "sm_plane_sampler_run_device": (C.c_int, [_VP, _VP, C.c_int64, C.c_int64, _VP, C.POINTER(C.c_int64), _VP, _VP]),
    "sm_plane_sampler_indices": (C.c_int, [_VP, _VP, C.POINTER(C.c_int64), _VP, C.POINTER(C.c_int64)]),
    "sm_plane_sampler_plane_indices": (C.c_int, [_VP, _VP, C.POINTER(C.c_int64)]),
    "sm_plane_sampler_last_error": (C.c_char_p, [_VP]),
    # include/sm_b200_debug.h (test hooks)
    "sm_debug_solve6": (C.c_int, [C.c_int, _VP, _VP, _VP, _VP]),
    "sm_debug_solve6_host": (C.c_int, [_VP, _VP, _VP, _VP]),
    "sm_debug_kabsch_host": (C.c_int, [_VP, _VP, _VP, _VP]),
    "sm_debug_bfgs_minimize": (C.c_int, [_VP, _VP, _VP, C.c_double, C.c_int32, _VP, _VP, _VP]),
    "sm_debug_ndt_newton": (C.c_int, [_VP, _VP, _VP, C.c_int32, C.c_float, C.c_double, C.c_double, C.c_double, C.c_int32,
                                      _VP, _VP, _VP, _VP]),
    "sm_debug_normals_leaf": (C.c_int, [_VP, C.c_int32, _VP, _VP, _VP]),
    "sm_debug_pm_surface_normal_leaf_host": (C.c_int, [_VP, C.c_int32, _VP, _VP, _VP, _VP]),
    "sm_debug_voxel_index": (C.c_int, [C.c_int32, _VP, C.c_float, C.c_int32, _VP]),
    "sm_debug_gicp_point": (C.c_int, [C.c_int32, _VP, _VP]),
    "sm_debug_gicp_outer": (C.c_int, [_VP, _VP, _VP, _VP, _VP, _VP, _VP]),
    "sm_debug_gicp_host": (C.c_int, [C.c_int32, _VP, _VP]),
    "sm_debug_motion_host": (C.c_int, [_VP, C.c_int64, _DP, _VP]),
    "sm_debug_inner_compensation_host": (C.c_int, [_DP, _VP, _VP, _VP, C.c_int64, _VP, _VP]),
    "sm_debug_icp_host": (C.c_int, [C.c_int32, _VP, C.c_int64, _VP]),
    "sm_debug_ndt_leaf": (C.c_int, [_VP, C.c_int32, C.c_int32, C.c_double, _VP, _VP, _VP, _VP, _VP]),
    "sm_debug_ndt_term": (C.c_int, [_VP, C.c_double, C.c_float, C.c_int32, _VP, _VP, _VP, _VP, _VP]),
    "sm_debug_ndt_host": (C.c_int, [C.c_int32, _VP, _VP]),
    "sm_debug_knn1_batched": (C.c_int, [C.c_int, _VP, C.c_int64, _VP, C.c_int64, C.c_double, C.c_int, C.c_int32, _VP, _VP]),
    "sm_debug_ndt_grid": (C.c_int, [C.c_int, _VP, C.c_int64, C.c_float, _VP, _VP, _VP, _VP, _VP, _VP, _VP, _VP]),
    "sm_debug_ndt_derivatives": (C.c_int, [C.c_int, _VP, C.c_int64, _VP, C.c_int64, C.c_float, C.c_double,
                                           C.c_int32, _VP, C.c_int32, _VP]),
    "sm_debug_ndt_derivatives_search": (C.c_int, [C.c_int, _VP, C.c_int64, _VP, C.c_int64, C.c_float, C.c_double,
                                                  C.c_int32, _VP, C.c_int32, _VP]),
    "sm_debug_ndt_direct_neighbors": (C.c_int, [C.c_int32, _VP, C.c_int64, C.c_float, _VP, _VP, _VP, _VP, C.c_int64,
                                                _VP, _VP]),
    "sm_debug_float_tree_knn": (C.c_int, [C.c_int, _VP, C.c_int64, _VP, C.c_int64, C.c_int32, _VP, _VP]),
    "sm_debug_pm_stages": (C.c_int, [C.c_int, _VP, C.c_int64, _VP, C.c_int64, C.c_float, C.c_uint32, _VP, C.c_float,
                                     C.c_float, _VP, _VP, _VP, _VP]),
    "sm_debug_pm_rand_window_host": (C.c_int, [C.c_uint32, C.c_int64, _VP]),
    "sm_debug_pm_rand_advance_host": (C.c_int, [_VP, C.c_uint64, _VP]),
    "sm_debug_pm_rand_draws_host": (C.c_int, [C.c_uint32, C.c_int64, C.c_int64, _VP]),
    "sm_debug_pm_rand_sample": (C.c_int, [C.c_int, _VP, C.c_int64, C.c_float, C.c_uint32, C.c_int64, _VP, _VP, _VP]),
    "sm_debug_pm_surface_normals": (C.c_int, [C.c_int, C.c_int32, _VP, C.c_int64, _VP, C.c_int64, _VP, _VP, _VP, _VP]),
    "sm_debug_icp_iteration": (C.c_int, [C.c_int, _VP, C.c_int64, _VP, _VP, C.c_int64, _VP, C.c_float, C.c_float,
                                         C.c_int32, C.c_int32, C.c_int32] + [_VP] * 16),
    "sm_debug_icp_iteration_minimizer": (C.c_int, [C.c_int, _VP, C.c_int64, _VP, _VP, C.c_int64, _VP, C.c_float,
                                                   C.c_float, C.c_int32, C.c_int32, C.c_int32, C.c_int32] + [_VP] * 16),
    "sm_debug_approx_voxel_grid": (C.c_int, [C.c_int, _VP, C.c_int64, C.c_float, _VP, _VP]),
    "sm_debug_gicp_covariances": (C.c_int, [C.c_int, _VP, C.c_int64, _VP]),
    "sm_debug_gicp_step": (C.c_int, [C.c_int, _VP, C.c_int64, _VP, C.c_int64, _VP, _VP, _VP, C.c_int32, _VP, _VP, _VP,
                                     _VP]),
    "sm_debug_m2dp_host": (C.c_int, [C.c_int32, _VP, _VP, _VP, C.c_int32, C.c_int32, _VP]),
    "sm_debug_m2dp_stages": (C.c_int, [C.c_int, _VP, C.c_int64, C.c_int64, C.c_double, C.c_double, C.c_int32,
                                       C.c_int32, C.c_int32, _VP, _VP, _VP, _VP, _VP, _VP, _VP, _VP]),
    "sm_debug_radix_sort": (C.c_int, [C.c_int, _VP, _VP, C.c_int64, C.c_int32, C.c_int64, C.c_int32, _VP, _VP]),
    "sm_debug_kd_tree": (C.c_int, [C.c_int, C.c_int32, C.c_int32, _VP, _VP, C.c_int64, _VP, _VP, C.c_int64, C.c_int32,
                                   _VP, _VP, _VP, _VP, _VP, _VP, _VP, _VP, _VP]),
    "sm_debug_filter_host": (C.c_int, [_VP, C.c_int32, C.c_int32, _VP, C.c_int64, _VP, _VP]),
    "sm_debug_filter_fit_host": (C.c_int, [_VP, _VP, C.c_int32, _VP]),
    "sm_debug_filter_distance_host": (C.c_int, [_VP, C.c_int32, C.c_float, C.c_float, _VP]),
    "sm_debug_mt19937_words_host": (C.c_int, [C.c_uint32, C.c_int64, _VP]),
    "sm_debug_filter_mt19937_flags": (C.c_int, [C.c_int, C.c_int64, C.c_float, C.c_uint32, _VP, C.POINTER(C.c_int64)]),
    "sm_debug_nth_element": (C.c_int, [C.c_int, _VP, C.c_int64, C.c_int64, _VP]),
    "sm_debug_normals_nth_perm": (C.c_int, [C.c_int, _VP, C.c_int64, _VP]),
    "sm_debug_voxel_bucket_counts_host": (C.c_int, [C.c_int64, _VP]),
    "sm_debug_voxel_hash_host": (C.c_int, [_VP, C.c_int64, _VP]),
    "sm_debug_voxel_unordered_epochs": (C.c_int, [C.c_int, _VP, C.c_int64, C.c_int64, C.c_float, _VP, _VP, _VP,
                                                  C.c_int64, C.POINTER(C.c_int64), C.POINTER(C.c_int32)]),
    "sm_debug_filter_ground_removal2": (C.c_int, [C.c_int, _VP, C.c_int32, _VP, C.c_int64, C.c_int64, C.c_int32, _VP, _VP,
                                                  _VP, _VP, _VP, _VP, _VP]),
    "sm_debug_depth_edge_host": (C.c_int, [_VP, C.c_int32, _VP, _VP, _VP, C.c_int64, _VP, _VP, _VP]),
    "sm_debug_depth_cluster": (C.c_int, [C.c_int, _VP, C.c_int32, _VP, C.c_int64, C.c_int64, _VP, _VP, _VP, _VP, _VP,
                                         _VP, _VP]),
    "sm_debug_statistic_removal_exact_sum_host": (C.c_int, [_VP, C.c_int64, _DP]),
    "sm_debug_statistic_removal_distance_host": (C.c_int, [_VP, _VP, C.c_int32, _VP]),
    "sm_debug_statistic_removal_distances": (C.c_int, [_VP, _VP, C.c_int64, C.POINTER(C.c_int64)]),
    "sm_debug_ground_removal_index_host": (C.c_int, [_VP, C.c_int64, C.c_int64, C.c_float, _VP]),
    "sm_debug_ground_removal_voxel_host": (C.c_int, [_VP, C.c_int64, C.c_int32, C.c_int32, C.c_float, _VP, _VP]),
    "sm_debug_plane_sampler_piece_host": (C.c_int, [C.c_int32, _VP, _VP]),
    "sm_debug_plane_sampler_keep_host": (C.c_int, [C.c_float, C.c_int64, C.c_int64, _VP]),
    "sm_debug_plane_sampler_trace": (C.c_int, [_VP, C.c_int32]),
    "sm_debug_plane_sampler_voxels": (C.c_int, [_VP, _VP, C.c_int64, C.POINTER(C.c_int64)]),
    "sm_lum_create": (C.c_int, [C.c_int, C.POINTER(_VP)]),
    "sm_lum_destroy": (C.c_int, [_VP]),
    "sm_lum_add_cloud": (C.c_int, [_VP, _VP, C.c_int64, C.c_int64, _VP]),
    "sm_lum_size": (C.c_int64, [_VP]),
    "sm_lum_align_all": (C.c_int, [_VP, _VP, C.c_int64, C.POINTER(C.c_int64)]),
    "sm_lum_poses": (C.c_int, [_VP, _VP, C.c_int64, C.POINTER(C.c_int64)]),
    "sm_lum_last_error": (C.c_char_p, [_VP]),
    "sm_debug_lum_correspondences": (C.c_int, [_VP, C.c_int32, C.c_int32, _VP, C.c_int64, C.POINTER(C.c_int64)]),
    "sm_debug_lum_trace": (C.c_int, [_VP, C.c_int32]),
    "sm_debug_lum_trace_get": (C.c_int, [_VP, C.c_int64, _IP, _IP, _VP, _VP, _VP, _DP]),
    "sm_device_count": (C.c_int, []),
    "sm_version": (C.c_char_p, []),
}


def lib():
    """Load libsm_b200.so; raise loudly if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; "
                "g.build()'` (nvcc, sm_90a).  staticmapping_b200 has no CPU fallback.")
        _lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(_lib, name)
            fn.restype = res
            fn.argtypes = args
    return _lib
