"""ctypes binding of libmorefusion_sm90a.so (include/morefusion_b200.h).

The CUDA library is the product: there is NO CPU or PyTorch fallback.  If the
shared library is missing or a call is made without a CUDA device, this module
raises -- it never silently routes elsewhere.
"""

import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libmorefusion_sm90a.so")

c_f, c_i, c_i64, c_p, c_sz = (ctypes.c_float, ctypes.c_int, ctypes.c_int64, ctypes.c_void_p,
                              ctypes.c_size_t)
c_d = ctypes.c_double
c_ll = ctypes.c_longlong

# name -> (restype, argtypes); must list every symbol the header declares
# (tests/test_abi.py cross-checks this table against include/morefusion_b200.h)
_geom = [c_f, c_f, c_f, c_f, c_i, c_i, c_i]      # origin xyz, pitch, X, Y, Z
_pgeom = [c_f, c_f, c_f, c_f, c_i, c_i, c_i]     # pitch, origin xyz, X, Y, Z
SIGNATURES = {
    "mf_abi_version": (c_i, []),
    "mf_device_sm_count": (c_i, [c_i]),
    "mf_average_voxelization_3d_workspace_bytes": (c_sz, [c_i64]),
    "mf_average_voxelization_3d_flags_offset": (c_sz, []),
    "mf_average_voxelization_3d_fwd": (c_i, [c_p, c_p, c_p, c_i64, c_i, c_i] + _geom + [c_p, c_p, c_p, c_sz, c_p, c_p]),
    "mf_debug_fill_probe": (c_i, [c_p, c_i, c_i, c_i64, c_i, c_p]),
    "mf_average_voxelization_3d_bwd": (c_i, [c_p, c_p, c_p, c_p, c_i64, c_i, c_i] + _geom + [c_p, c_p]),
    "mf_max_voxelization_3d_workspace_bytes": (c_sz, [c_i, c_i, c_i, c_i]),
    "mf_max_voxelization_3d_fwd": (c_i, [c_p, c_p, c_p, c_p, c_i64, c_i, c_i] + _geom + [c_p, c_p, c_p, c_sz, c_p, c_p]),
    "mf_max_voxelization_3d_bwd": (c_i, [c_p, c_p, c_i64, c_i, c_i, c_i, c_i, c_i, c_p, c_p]),
    "mf_interpolate_voxel_grid_fwd": (c_i, [c_p, c_p, c_p, c_i64, c_i, c_i, c_i, c_i, c_i, c_i, c_p, c_p]),
    "mf_interpolate_voxel_grid_bwd": (c_i, [c_p, c_p, c_p, c_i64, c_i, c_i, c_i, c_i, c_i, c_i, c_p, c_p]),
    "mf_interpolate_voxel_grid_path": (c_i, [c_i64, c_i, c_i, c_i, c_i, c_i, c_i, c_i, c_i, c_p]),
    "mf_truncated_distance_function_workspace_bytes": (c_sz, [c_i, c_i, c_i]),
    "mf_truncated_distance_function_fwd": (c_i, [c_p, c_i64] + _pgeom + [c_f, c_p, c_p, c_p, c_sz, c_p]),
    "mf_truncated_distance_function_bwd": (c_i, [c_p, c_p, c_p, c_i64] + _pgeom + [c_f, c_p, c_p]),
    "mf_pseudo_occupancy_voxelization_workspace_bytes": (c_sz, [c_i, c_i, c_i]),
    "mf_pseudo_occupancy_voxelization_fwd": (c_i, [c_p, c_p, c_i64] + _pgeom + [c_f, c_f] + [c_p] * 7 + [c_p, c_sz, c_p]),
    "mf_occupancy_grid_3d_fwd": (c_i, [c_p, c_i64] + _pgeom + [c_f, c_p, c_p, c_p]),
    "mf_occupancy_grid_3d_bwd": (c_i, [c_p, c_p, c_p, c_i64] + _pgeom + [c_f, c_p, c_p]),
    "mf_quaternion_matrix_fwd": (c_i, [c_p, c_i64, c_p, c_p]),
    "mf_quaternion_matrix_bwd": (c_i, [c_p, c_p, c_i64, c_p, c_p]),
    "mf_compose_transform_fwd": (c_i, [c_p, c_p, c_i64, c_p, c_p]),
    "mf_transform_points_fwd": (c_i, [c_p, c_i64, c_p, c_i64, c_p, c_p]),
    "mf_transform_points_bwd": (c_i, [c_p, c_p, c_i64, c_p, c_i64, c_p, c_p, c_p]),
    "mf_cnn_point_mlp": (c_i, [c_p] * 10 + [c_i, c_i, c_f, c_p, c_i, c_p, c_p]),
    "mf_cnn_point_mlp_voxkeys": (c_i, [c_p] * 10 + [c_i, c_i, c_f, c_p, c_i, c_p, c_i, c_i, c_i, c_p, c_p, c_p]),
    "mf_cnn_occ_convs": (c_i, [c_p] * 5 + [c_i, c_i, c_p, c_p, c_p, c_i, c_i, c_p]),
    "mf_cnn_occ_convs_tc": (c_i, [c_p] * 5 + [c_i, c_i, c_p, c_p, c_i, c_i, c_p]),
    "mf_cnn_voxelize_s2d": (c_i, [c_p, c_p, c_i, c_i, c_i, c_i, c_i, c_p, c_p, c_p]),
    "mf_cnn_voxelize_s2d_phase": (c_i, [c_p, c_p, c_i, c_i, c_i, c_i, c_i, c_p, c_p, c_i, c_p]),
    "mf_cnn_occ_convs_tc_u8": (c_i, [c_p] * 5 + [c_i, c_i, c_p, c_p, c_i, c_i, c_p]),
    "mf_cnn_occ_fused": (c_i, [c_p] * 5 + [c_i, c_i, c_p, c_i, c_i, c_p]),
    "mf_cnn_occ_fused_u8": (c_i, [c_p] * 5 + [c_i, c_i, c_p, c_i, c_i, c_p]),
    "mf_cnn_pack_s2d": (c_i, [c_p, c_p, c_i, c_i, c_i, c_i, c_p, c_p]),
    "mf_gemm_bf16_simt": (c_i, [c_p, c_p]),
    "mf_gemm_bf16_tc_workspace_bytes": (c_sz, [c_i, c_i]),
    "mf_gemm_bf16_tc": (c_i, [c_p, c_p, c_sz, c_p]),
    "mf_gemm_bf16_tc_ex": (c_i, [c_p, c_i, c_p, c_sz, c_p, c_p, c_i, c_p]),
    "mf_gemm_bf16_tc_plan": (c_i, [c_p, c_i, c_sz, c_i, c_i, c_i, c_i, c_p]),
    "mf_gemm_bf16_tc_pair_clusters": (c_i, [c_i, c_p]),
    "mf_gemm_bf16_tc_segments": (c_i, [c_i, c_i, c_i, c_p, c_i]),
    "mf_cnn_heads_tc": (c_i, [c_p, c_i, c_p, c_p]),
    "mf_gemm_bf16_simt_grouped": (c_i, [c_p, c_i, c_p]),
    "mf_gemm_bf16_tc_grouped": (c_i, [c_p, c_i, c_p, c_sz, c_p]),
    "mf_cnn_interp_cl": (c_i, [c_p, c_i, c_p, c_i, c_i, c_i, c_i, c_f, c_p, c_i, c_i, c_p]),
    "mf_cnn_pose": (c_i, [c_p] * 7 + [c_i, c_i, c_i, c_p, c_p, c_p, c_p]),
    "mf_cnn_head4_pose": (c_i, [c_p, c_i] + [c_p] * 10 + [c_i, c_i, c_i, c_p, c_p, c_p, c_p]),
    "mf_posenet_point_mlp": (c_i, [c_p] * 11 + [c_i, c_i, c_p, c_i, c_p, c_p]),
    "mf_posenet_pool": (c_i, [c_p, c_i, c_i, c_i, c_p, c_p]),
    "mf_posenet_obj_bias": (c_i, [c_p, c_ll, c_i, c_i, c_p, c_p, c_i, c_p, c_p]),
    "mf_posenet_obj_bias_bwd": (c_i, [c_p, c_p, c_p, c_ll, c_i, c_i, c_i, c_p, c_ll, c_p, c_p, c_p]),
    "mf_posenet_obj_colsum": (c_i, [c_p, c_ll, c_i, c_i, c_i, c_p, c_p]),
    "mf_posenet_pool_bwd": (c_i, [c_p, c_p, c_i, c_i, c_i, c_p, c_p]),
    "mf_posenet_point_mlp_bwd": (c_i, [c_p] * 10 + [c_i, c_i] + [c_p] * 12),
    "mf_cnn_point_mlp_f32": (c_i, [c_p] * 10 + [c_i, c_i, c_f, c_p, c_i, c_p, c_p, c_p]),
    "mf_px_split": (c_i, [c_p, c_ll, c_ll, c_i, c_p, c_p, c_ll, c_i, c_p]),
    "mf_px_combine": (c_i, [c_p, c_i, c_ll, c_i, c_p, c_i, c_i, c_i, c_p, c_p, c_ll, c_i, c_p]),
    "mf_px_pack_s2d": (c_i, [c_p, c_p, c_i, c_i, c_i, c_i, c_p, c_p, c_p]),
    "mf_px_interp": (c_i, [c_p, c_p, c_i, c_p, c_i, c_i, c_i, c_i, c_f, c_p, c_p, c_i, c_i, c_p]),
    "mf_px_head4_pose": (c_i, [c_p, c_p, c_i] + [c_p] * 10 + [c_i, c_i, c_i, c_p, c_p, c_p, c_p]),
    "mf_cnn_head4_pose_train": (c_i, [c_p, c_i] + [c_p] * 10 + [c_i, c_i, c_i, c_p, c_p, c_p, c_p, c_p]),
    "mf_train_gemm_tn": (c_i, [c_p, c_ll, c_p, c_ll, c_i, c_i, c_i, c_p, c_ll, c_i, c_ll, c_ll, c_ll, c_i, c_p]),
    "mf_train_conv_wgrad": (c_i, [c_p, c_p, c_i, c_i, c_i, c_i, c_p, c_i, c_p]),
    "mf_train_conv_dgrad": (c_i, [c_p, c_p, c_i, c_i, c_i, c_i, c_i, c_p, c_ll, c_ll, c_p]),
    "mf_train_head4_bwd": (c_i, [c_p] * 5 + [c_i] + [c_p] * 5 + [c_i, c_i, c_i] + [c_p] * 8),
    "mf_train_relu_mask": (c_i, [c_p, c_ll, c_p, c_ll, c_ll, c_i, c_p]),
    "mf_train_colsum": (c_i, [c_p, c_ll, c_ll, c_i, c_p, c_p]),
    "mf_train_interp_bwd": (c_i, [c_p, c_ll, c_i, c_p, c_i, c_i, c_i, c_i, c_f, c_p, c_p]),
    "mf_train_mask_pack": (c_i, [c_p, c_p, c_i, c_i, c_i, c_i, c_p, c_p, c_p]),
    "mf_train_vox_bwd": (c_i, [c_p, c_ll, c_p, c_i, c_i, c_i, c_i, c_p, c_ll, c_i, c_p, c_p]),
    "mf_train_point_mlp_bwd": (c_i, [c_p, c_p, c_p, c_ll, c_p, c_ll] + [c_p] * 6 + [c_i, c_i, c_f] + [c_p] * 10),
    "mf_train_adam": (c_i, [c_p, c_p, c_p, c_p, c_i64, c_f, c_d, c_d, c_d, c_d, c_f, c_p]),
    "mf_pointcloud_from_depth": (c_i, [c_p, c_i, c_i, c_f, c_f, c_f, c_f, c_i, c_p, c_p]),
    "mf_masks_to_bboxes": (c_i, [c_p, c_i, c_i, c_i, c_p, c_p]),
    "mf_label_bboxes_workspace_bytes": (c_sz, [c_i]),
    "mf_label_bboxes": (c_i, [c_p, c_p, c_i, c_i, c_p, c_i, c_i, c_i, c_p, c_p, c_sz, c_p]),
    "mf_instance_crops": (c_i, [c_p, c_p, c_p, c_i, c_i, c_p, c_p, c_i, c_i, c_p, c_p, c_p]),
    "mf_psp_tail_sampled": (c_i, [c_p, c_p, c_i, c_i, c_i, c_i, c_p, c_p, c_p, c_p, c_p, c_p, c_p]),
    "mf_map_integrate": (c_i, [c_p, c_p, c_i64, c_f, c_f, c_f, c_d, c_i, ctypes.c_uint32, c_f, c_f, c_f, c_f,
                                c_p, c_p, c_i64, c_p, c_p]),
    "mf_map_integrate_labelled": (c_i, [c_p, c_p, c_i64, c_f, c_f, c_f, c_p, c_i, c_i, c_p, ctypes.c_uint32,
                                         c_f, c_f, c_f, c_f, c_p, c_p, c_i64, c_p, c_p]),
    "mf_map_update_points": (c_i, [c_p, c_i64, c_d, c_i, c_f, c_f, c_f, c_p, c_p, c_i64, c_p, c_p]),
    "mf_map_query_grids": (c_i, [c_p, c_p, c_p, c_i, c_i, c_i, c_i, c_p, c_i, c_p, c_p, c_i64, c_p,
                                  c_p, c_p, c_p, c_p]),
    "mf_map_query_node_grids": (c_i, [c_p, c_p, c_p, c_i, c_i, c_i, c_i, c_p, c_p, c_i, c_i, c_d,
                                       c_p, c_p, c_i64, c_p, c_p, c_p, c_p]),
    "mf_map_query_node_grids_world": (c_i, [c_p, c_p, c_p, c_i, c_i, c_i, c_i, c_p, c_p, c_i, c_i, c_d,
                                             c_p, c_i, c_p, c_p, c_i64, c_p, c_p, c_p, c_p]),
    "mf_map_integrate_server": (c_i, [c_p, c_p, c_i, c_i, c_p, c_d, c_p, c_i, c_i, c_p, c_i, c_i, c_d,
                                       c_i, ctypes.c_uint32, c_f, c_f, c_f, c_f, c_p, c_p, c_p, c_p,
                                       c_p, c_p, c_i64, c_p, c_p, c_p, c_p]),
    "mf_map_render": (c_i, [c_p, c_i, c_i, c_p, c_f, c_f, c_f, c_f, c_p, c_p, c_i, c_p, c_p, c_i,
                            c_p, c_p, c_p, c_p, c_p, c_i64, c_p, c_p]),
    "mf_map_server_grid_params": (c_i, [c_p, c_i, c_p, c_p, c_p, c_d, c_d, c_d, c_p, c_p, c_p]),
    "mf_objmap_state_bytes": (c_sz, [c_i]),
    "mf_objmap_append": (c_i, [c_p, c_i, c_p, c_i, c_p, c_p, c_p, c_p, c_i, c_p]),
    "mf_objmap_vote": (c_i, [c_p, c_i, c_p, c_i, c_i, c_p, c_i, c_p, c_i64, c_p]),
    "mf_objmap_remove": (c_i, [c_p, c_i, c_p, c_i, c_p]),
    "mf_objmap_reset": (c_i, [c_p, c_i, c_p]),
    "mf_map_rehash": (c_i, [c_p, c_i64, c_p, c_p, c_i64, c_p, c_p]),
    "mf_icc_max_group_size": (c_i, [c_i]),
    "mf_icc_workspace_bytes": (c_sz, [c_i, c_i, c_i, c_i, c_i]),
    "mf_icc_run": (c_i, [c_i, c_i, c_i, c_f, c_f] + [c_p] * 7 + [c_i] + [c_p] * 9
                   + [c_i, c_i, c_p, c_p, c_d, c_d, c_d, c_d, c_p, c_p, c_i, c_p, c_sz, c_p]),
    "mf_average_distance_fwd": (c_i, [c_p, c_i, c_p, c_p, c_i, c_i, c_p, c_p, c_p]),
    "mf_average_distance_fwd_parts": (c_i, [c_p, c_i, c_p, c_p, c_i, c_i, c_i, c_p, c_p, c_p]),
    "mf_average_distance_bwd": (c_i, [c_p, c_p, c_i, c_p, c_p, c_i, c_p, c_p, c_p, c_p, c_p]),
    "mf_average_distance_fwd_batched": (c_i, [c_p, c_i, c_p, c_p, c_i, c_i, c_p, c_p, c_p, c_p]),
    "mf_average_distance_bwd_batched": (c_i, [c_p, c_p, c_i, c_p, c_p, c_i, c_i, c_p, c_p, c_p, c_p, c_p, c_p]),
    "mf_icc_run_profiled": (c_i, [c_i, c_i, c_i, c_f, c_f] + [c_p] * 7 + [c_i] + [c_p] * 9
                            + [c_i, c_i, c_p, c_p, c_d, c_d, c_d, c_d, c_p, c_p, c_i, c_p, c_sz, c_p, c_p]),
    "mf_icc_observer_state_bytes": (c_sz, [c_i]),
    "mf_icc_run_early_stop": (c_i, [c_i, c_i, c_i, c_f, c_f] + [c_p] * 7 + [c_i] + [c_p] * 9
                              + [c_i, c_i, c_p, c_p, c_d, c_d, c_d, c_d, c_p, c_p, c_i, c_p, c_sz, c_p]
                              + [c_p, c_sz, c_d, c_i, c_i, c_p, c_p]),
    "mf_icp_sort_workspace_bytes": (c_sz, [c_i, c_i]),
    "mf_icp_voxel_down_sample": (c_i, [c_p, c_i, c_i, c_i, c_d, c_p, c_p, c_p, c_p, c_p, c_sz, c_p]),
    "mf_icp_cell_list": (c_i, [c_p, c_p, c_i, c_d, c_p, c_p, c_p, c_p, c_p, c_sz, c_p]),
    "mf_icp_run_workspace_bytes": (c_sz, [c_i, c_i]),
    "mf_icp_run": (c_i, [c_i, c_p, c_i, c_p, c_p, c_p, c_p, c_d, c_i, c_d, c_d, c_p, c_p, c_p, c_p,
                         c_p, c_sz, c_p]),
    "mf_occupancy_registration_workspace_bytes": (c_sz, [c_i, c_i, c_i, c_i]),
    "mf_occupancy_registration_run": (c_i, [c_i, c_p, c_i, c_p, c_p, c_i, c_i, c_i, c_i, c_p, c_p, c_p,
                                            c_f, c_p, c_p, c_i, c_d, c_p, c_p, c_p, c_p, c_p, c_sz,
                                            c_p]),
    "mf_icp_link_workspace_bytes": (c_sz, [c_i, c_i]),
    "mf_icp_link_cluster_size": (c_i, [c_i]),
    "mf_icp_link_run": (c_i, [c_i, c_p, c_i, c_p, c_p, c_i, c_p, c_p, c_p, c_i, c_i, c_p, c_p, c_p,
                              c_p, c_p, c_p, c_p, c_i, c_p, c_sz, c_p]),
    "mf_pose_metrics_workspace_bytes": (c_sz, [c_i]),
    "mf_pose_metrics": (c_i, [c_i, c_p, c_p, c_p, c_p, c_p, c_i, c_p, c_i, c_p, c_sz, c_p, c_p]),
    "mf_training_full_grids": (c_i, [c_i, c_p, c_p, c_p, c_i, c_p, c_p, c_p, c_p, c_p, c_p]),
    "mf_training_nontarget_present": (c_i, [c_i, c_p, c_p, c_p]),
    "mf_training_transform": (c_i, [c_i, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p]),
    "mf_render_cad_workspace_bytes": (c_sz, [c_i, c_i, c_i, c_i]),
    "mf_render_cad": (c_i, [c_p, c_i, c_p, c_i, c_p, c_i, c_p, c_p, c_i, c_d, c_i, c_i, c_p, c_p,
                            c_p, c_p, c_sz, c_p]),
    "mf_render_scene": (c_i, [c_p, c_i, c_p, c_i, c_p, c_i, c_p, c_p, c_p, c_i, c_d, c_i, c_i, c_p,
                              c_p, c_p, c_p, c_p, c_sz, c_p]),
    "mf_mesh_voxelize_workspace_bytes": (c_sz, [c_i, c_i]),
    "mf_mesh_voxelize_solid": (c_i, [c_p, c_i, c_p, c_i, c_p, c_i, c_i, c_p, c_p, c_p, c_p, c_p, c_p,
                                     c_p, c_sz, c_p]),
    "mf_mesh_signed_distance_workspace_bytes": (c_sz, [c_i, c_i]),
    "mf_mesh_signed_distance": (c_i, [c_p, c_i, c_p, c_i, c_p, c_i, c_p, c_p, c_i, c_p, c_p, c_p,
                                      c_sz, c_p]),
}

_lib = None


class LibraryMissing(RuntimeError):
    pass


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise LibraryMissing(
                f"{LIB_PATH} not built; run `python -m morefusion_b200.build` "
                "(morefusion_b200 has no CPU fallback)")
        L = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


_ERR = {-1: "invalid argument", -2: "problem too large for int32 keys",
        -3: "workspace too small", -4: "unsupported shape"}


def check(rc, what=""):
    if rc == 0:
        return
    if rc < 0:
        raise ValueError(f"{what}: {_ERR.get(rc, rc)}")
    raise RuntimeError(f"{what}: CUDA error {rc}")


def ptr(t):
    if t is None:
        return None
    return ctypes.c_void_p(t.data_ptr())


def stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise RuntimeError(
                "morefusion_b200 operators run on CUDA tensors only (no CPU fallback); "
                f"got a tensor on {t.device}")
