"""ctypes binding of the C ABI declared in include/pvraft_b200.h.

The shared library is mandatory: importing the package never falls back to PyTorch ops or to the
CPU oracle -- a missing/unbuildable `libpvraft_b200.so` raises at first use.
"""
import ctypes as C
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libpvraft_b200.so')

c_float_p = C.POINTER(C.c_float)
c_double_p = C.POINTER(C.c_double)
c_int32_p = C.POINTER(C.c_int32)
c_int8_p = C.POINTER(C.c_int8)
VP = C.c_void_p   # device pointers travel as plain addresses

IN_PLAIN, IN_GN, IN_GN_MINMAX = 0, 1, 2
ACT_NONE, ACT_RELU, ACT_LRELU = 0, 1, 2
KNN = 32
MOMENTS = 16


class LinearArgs(C.Structure):
    _fields_ = [('in_', VP), ('in_min', VP), ('in_stats', VP), ('in_gamma', VP), ('in_beta', VP),
                ('in_count', C.c_double), ('in_mode', C.c_int), ('in_act', C.c_int), ('in_slope', C.c_float),
                ('weight', VP), ('w_ld', C.c_int), ('w_cin', C.c_int), ('bias', VP), ('residual', VP), ('out_act', C.c_int),
                ('out', VP), ('out_stats', VP), ('B', C.c_int), ('N', C.c_int), ('cin', C.c_int), ('cout', C.c_int)]


class TcLinearArgs(C.Structure):
    _fields_ = [('in_', VP * 3), ('in_channels', C.c_int * 3), ('in_min', VP), ('in_stats', VP), ('in_gamma', VP),
                ('in_beta', VP), ('in_count', C.c_double), ('in_act', C.c_int), ('in_slope', C.c_float), ('w_hi', VP),
                ('w_lo', VP), ('n_pad', C.c_int), ('cout', C.c_int), ('bias', VP), ('bias2', VP), ('out_act', C.c_int),
                ('residual', VP), ('out', VP), ('out2', VP), ('h', VP), ('z', VP), ('out_stats', VP), ('epilogue', C.c_int),
                ('B', C.c_int), ('N', C.c_int), ('tail', VP), ('w3', VP), ('b3', VP), ('coords1', VP), ('coords2', VP),
                ('coords2_out', VP), ('flow_out', VP), ('params_settled', C.c_int), ('w_bf16', VP)]


class UpdateChainArgs(C.Structure):
    _fields_ = [('y1', VP), ('y1_stats', VP), ('gn_gamma', VP), ('gn_beta', VP), ('gn_count', C.c_double),
                ('gn_slope', C.c_float), ('kfeat', VP), ('cflow', VP), ('flow', VP), ('net', VP), ('inp', VP),
                ('w_hi', VP * 5), ('w_lo', VP * 5), ('b_cc', VP), ('b_m', VP), ('b_z', VP), ('b_r', VP), ('b_q', VP),
                ('net_out', VP), ('p_out', VP), ('B', C.c_int), ('N', C.c_int), ('hidden', C.c_int), ('context', C.c_int),
                ('y1_channels', C.c_int), ('w_bf16', VP * 5)]


class KnnBranchArgs(C.Structure):
    _fields_ = [('knn_sel', VP), ('moments', VP), ('w_knn', VP), ('b_knn', VP), ('gnk_gamma', VP), ('gnk_beta', VP),
                ('preluk', VP), ('preluk_host', C.c_float), ('kfeat', VP), ('flow', VP), ('w_cf', VP), ('b_cf', VP),
                ('cflow', VP), ('B', C.c_int), ('N', C.c_int)]


class CorrFeatArgs(C.Structure):
    _fields_ = [('y1', VP), ('y1_stats', VP), ('gn1_gamma', VP), ('gn1_beta', VP), ('prelu1', VP), ('w_out', VP),
                ('b_out', VP), ('knn_sel', VP), ('moments', VP), ('w_knn', VP), ('b_knn', VP), ('gnk_gamma', VP),
                ('gnk_beta', VP), ('preluk', VP), ('w_kout', VP), ('b_kout', VP), ('corr_feat', VP), ('corr_in', VP),
                ('flow', VP), ('w_cc', VP), ('b_cc', VP), ('w_cf', VP), ('b_cf', VP), ('w_cm', VP), ('b_cm', VP),
                ('motion', VP), ('B', C.c_int), ('N', C.c_int)]


class GruArgs(C.Structure):
    _fields_ = [('net', VP), ('inp', VP), ('motion', VP), ('w_z', VP), ('b_z', VP), ('w_r', VP), ('b_r', VP),
                ('w_q', VP), ('b_q', VP), ('net_out', VP), ('B', C.c_int), ('N', C.c_int)]


class FlowOutArgs(C.Structure):
    _fields_ = [('z3', VP), ('z3_stats', VP), ('gn3_gamma', VP), ('gn3_beta', VP), ('net', VP), ('w_c1', VP),
                ('b_c1', VP), ('w_o0', VP), ('b_o0', VP), ('w_o2', VP), ('b_o2', VP), ('coords1', VP),
                ('coords2', VP), ('delta', VP), ('coords2_out', VP), ('flow_out', VP), ('B', C.c_int), ('N', C.c_int)]


_SIGNATURES = {
    'pvraft_version': (C.c_int, []),
    'pvraft_last_error_string': (C.c_char_p, []),
    'pvraft_device_info': (C.c_int, [C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    'pvraft_corr_matmul_workspace_bytes': (C.c_int64, [C.c_int, C.c_int, C.c_int, C.c_int]),
    'pvraft_corr_matmul_fwd': (C.c_int, [VP, VP, C.c_int, C.c_int, C.c_int, C.c_int, VP, VP, VP]),
    'pvraft_tf32_split_fwd': (C.c_int, [VP, C.c_int64, VP, VP, VP]),
    'pvraft_corr_matmul_window_fwd': (C.c_int, [VP, VP, VP, VP, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                                C.c_int, VP, C.c_int64, VP]),
    'pvraft_corr_topk_fwd': (C.c_int, [VP, C.c_int, C.c_int, C.c_int, C.c_int, VP, VP, VP]),
    'pvraft_corr_topk_window_fwd': (C.c_int, [VP, C.c_int, C.c_int, C.c_int64, C.c_int, C.c_int, VP, VP, VP, C.c_int64, VP]),
    'pvraft_corr_reorder': (C.c_int, [VP, VP, C.c_int64, C.c_int, VP, VP, VP]),
    'pvraft_xyz_pad_fwd': (C.c_int, [VP, C.c_int64, VP, VP]),
    'pvraft_corr_lookup_fwd': (C.c_int, [VP, VP, VP, VP, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float,
                                         VP, C.c_int, VP, VP, VP, VP, VP, VP]),
    'pvraft_corr_lookup_bf16_fwd': (C.c_int, [VP, VP, VP, VP, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float,
                                              VP, C.c_int, VP, VP, VP, VP, VP, VP]),
    'pvraft_corr_lookup_det_workspace_bytes': (C.c_int64, [C.c_int]),
    'pvraft_corr_lookup_table_in_smem': (C.c_int, [C.c_int, C.c_int]),
    'pvraft_corr_state_pack_bf16': (C.c_int, [VP, VP, C.c_int64, VP, VP, VP]),
    'pvraft_linear_fwd': (C.c_int, [C.POINTER(LinearArgs), VP, VP]),
    'pvraft_linear_det_workspace_bytes': (C.c_int64, [C.c_int]),
    'pvraft_tc_linear_fwd': (C.c_int, [C.POINTER(TcLinearArgs), VP, VP]),
    'pvraft_tc_linear_det_workspace_bytes': (C.c_int64, [C.c_int]),
    'pvraft_update_chain_fwd': (C.c_int, [C.POINTER(UpdateChainArgs), VP]),
    'pvraft_tc_weight_split':(C.c_int, [VP, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, VP, VP, VP]),
    'pvraft_tc_weight_bf16': (C.c_int, [VP, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, VP, VP]),
    'pvraft_gn_act_fwd': (C.c_int, [VP, VP, VP, VP, C.c_double, C.c_int, C.c_float, C.c_int, C.c_int, C.c_int,
                                    C.c_int, VP, VP, VP]),
    'pvraft_corr_feature_fwd': (C.c_int, [C.POINTER(CorrFeatArgs), VP]),
    'pvraft_knn_branch_fwd': (C.c_int, [C.POINTER(KnnBranchArgs), VP]),
    'pvraft_point_order_fwd': (C.c_int, [VP, C.c_int, C.c_int, VP, VP, VP]),
    'pvraft_gru_fwd': (C.c_int, [C.POINTER(GruArgs), VP]),
    'pvraft_setconv_edge_fwd': (C.c_int, [VP, VP, VP, VP, C.c_int, C.c_int, C.c_int, C.c_int, VP, VP, VP, VP, VP, VP, VP]),
    'pvraft_setconv_edge_det_workspace_bytes': (C.c_int64, [C.c_int]),
    'pvraft_edge_plan_fwd': (C.c_int, [VP, VP, C.c_int, C.c_int, VP, VP]),
    'pvraft_edge_plan_bytes': (C.c_int64, [C.c_int, C.c_int]),
    'pvraft_flow_out_fwd': (C.c_int, [C.POINTER(FlowOutArgs), VP]),
    'pvraft_knn_workspace_bytes': (C.c_int64, [C.c_int, C.c_int]),
    'pvraft_knn_fwd': (C.c_int, [VP, VP, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, VP, VP, VP, VP]),
    'pvraft_linear_wgrad': (C.c_int, [VP, VP, C.c_int64, C.c_int, C.c_int, VP, C.c_int, VP, VP, VP]),
    'pvraft_linear_wgrad_det_workspace_bytes': (C.c_int64, [C.c_int, C.c_int]),
    'pvraft_tc_wgrad_bf16': (C.c_int, [VP, VP, C.c_int64, C.c_int, C.c_int, VP, C.c_int, VP, VP, VP]),
    'pvraft_tc_wgrad_bf16_det_workspace_bytes': (C.c_int64, [C.c_int, C.c_int]),
    'pvraft_gn_act_bwd': (C.c_int, [VP, VP, VP, VP, VP, C.c_double, C.c_int, C.c_float, C.c_int, C.c_int64, C.c_int, VP, VP, VP, VP,
                                    VP, VP, VP, VP, VP]),
    'pvraft_gn_act_bwd_det_workspace_bytes': (C.c_int64, [C.c_int, C.c_int]),
    'pvraft_linear_bwd_small': (C.c_int, [VP, VP, VP, C.c_int64, C.c_int, C.c_int, C.c_int, VP, C.c_int, VP, VP, VP, VP]),
    'pvraft_linear_bwd_small_det_workspace_bytes': (C.c_int64, [C.c_int, C.c_int]),
    'pvraft_gn_act_maxk_fwd': (C.c_int, [VP, VP, VP, VP, C.c_double, C.c_int, C.c_float, C.c_int, C.c_int64, C.c_int, VP, VP, VP, VP]),
    'pvraft_edge_fwd': (C.c_int, [VP, VP, VP, C.c_int, C.c_int, C.c_int, VP, VP, VP]),
    'pvraft_edge_fwd_det_workspace_bytes': (C.c_int64, [C.c_int]),
    'pvraft_edge_bwd': (C.c_int, [VP, VP, C.c_int, C.c_int, C.c_int, VP, VP, VP]),
    'pvraft_edge_bwd_det_workspace_bytes': (C.c_int64, [C.c_int, C.c_int, C.c_int]),
    'pvraft_maxk_fwd': (C.c_int, [VP, C.c_int64, C.c_int, VP, VP, VP]),
    'pvraft_maxk_bwd': (C.c_int, [VP, VP, C.c_int64, C.c_int, VP, VP]),
    'pvraft_corr_lookup_bwd': (C.c_int, [VP, VP, VP, VP, VP, C.c_int, VP, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float,
                                         VP, VP]),
    'pvraft_corr_lookup_xyz_bwd': (C.c_int, [VP, VP, VP, C.c_int, C.c_int, C.c_int, C.c_int, VP, VP, VP]),
    'pvraft_corr_lookup_xyz_bwd_det_workspace_bytes': (C.c_int64, [C.c_int, C.c_int]),
    'pvraft_corr_init_bwd': (C.c_int, [VP, VP, VP, VP, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, VP, VP, VP, VP]),
    'pvraft_corr_init_bwd_det_workspace_bytes': (C.c_int64, [C.c_int, C.c_int, C.c_int]),
    'pvraft_flow_metrics_fwd': (C.c_int, [VP, VP, VP, C.c_int64, VP, VP, VP]),
    'pvraft_flow_metrics_det_workspace_bytes': (C.c_int64, []),
    'pvraft_flow_l1_bwd': (C.c_int, [VP, VP, VP, C.c_int64, VP, VP, C.c_float, VP, VP]),
    'pvraft_chamfer_fwd': (C.c_int, [VP, VP, C.c_int, C.c_int, C.c_int, C.c_int, VP, VP, VP, VP, VP]),
    'pvraft_chamfer_fwd_det_workspace_bytes': (C.c_int64, [C.c_int]),
    'pvraft_chamfer_bwd': (C.c_int, [VP, VP, VP, VP, VP, C.c_int, C.c_int, C.c_int, C.c_int, VP, VP, VP, VP]),
    'pvraft_chamfer_bwd_det_workspace_bytes': (C.c_int64, [C.c_int, C.c_int, C.c_int, C.c_int]),
    'pvraft_flow_smooth_fwd': (C.c_int, [VP, VP, C.c_int, C.c_int, C.c_int, C.c_int, VP, VP, VP]),
    'pvraft_flow_smooth_fwd_det_workspace_bytes': (C.c_int64, [C.c_int]),
    'pvraft_flow_smooth_bwd': (C.c_int, [VP, VP, VP, C.c_int, C.c_int, C.c_int, C.c_int, VP, VP, VP]),
    'pvraft_flow_smooth_bwd_det_workspace_bytes': (C.c_int64, [C.c_int, C.c_int]),
    'pvraft_cloud_laplacian_fwd': (C.c_int, [VP, VP, C.c_int, C.c_int, C.c_int, VP, VP]),
    'pvraft_cloud_laplacian_bwd': (C.c_int, [VP, VP, C.c_int, C.c_int, C.c_int, VP, VP, VP]),
    'pvraft_cloud_laplacian_bwd_det_workspace_bytes': (C.c_int64, [C.c_int, C.c_int]),
    'pvraft_laplacian_fwd': (C.c_int, [VP, VP, VP, VP, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, VP, VP, VP, VP, VP]),
    'pvraft_laplacian_fwd_det_workspace_bytes': (C.c_int64, [C.c_int]),
    'pvraft_laplacian_bwd': (C.c_int, [VP, VP, VP, VP, VP, VP, VP, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, VP, VP, VP, VP,
                                       VP]),
    'pvraft_laplacian_bwd_det_workspace_bytes': (C.c_int64, [C.c_int, C.c_int, C.c_int, C.c_int]),
    'pvraft_flow_propagate_fwd':(C.c_int, [VP, VP, VP, C.c_int, C.c_int, C.c_int, C.c_int, VP, VP, VP]),
    'pvraft_flow_propagate_grid_fwd': (C.c_int, [VP, VP, VP, C.c_int, C.c_int, C.c_int, C.c_int, VP, VP, VP, VP]),
    'pvraft_grid_index_workspace_bytes': (C.c_int64, [C.c_int, C.c_int]),
    'pvraft_grid_index_fwd': (C.c_int, [VP, VP, C.c_int, C.c_int, VP, VP]),
    'pvraft_chamfer_grid_workspace_bytes': (C.c_int64, [C.c_int, C.c_int, C.c_int, C.c_int]),
    'pvraft_chamfer_grid_fwd': (C.c_int, [VP, VP, C.c_int, C.c_int, C.c_int, C.c_int, VP, VP, VP, VP, VP, VP]),
    'pvraft_laplacian_grid_fwd': (C.c_int, [VP, VP, VP, VP, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, VP, VP, VP, VP, VP,
                                            VP]),
    'pvraft_flow_consistency_fwd': (C.c_int, [VP, VP, VP, VP, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, VP, VP,
                                              VP, VP, VP, VP]),
    'pvraft_flow_consistency_fwd_det_workspace_bytes': (C.c_int64, [C.c_int]),
    'pvraft_flow_consistency_grid_fwd': (C.c_int, [VP, VP, VP, VP, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, VP,
                                                   VP, VP, VP, VP, VP, VP]),
    'pvraft_flow_consistency_bwd': (C.c_int, [VP, VP, VP, VP, VP, VP, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, VP, VP, VP, VP, VP,
                                              VP]),
    'pvraft_flow_consistency_bwd_det_workspace_bytes': (C.c_int64, [C.c_int, C.c_int, C.c_int]),
    'pvraft_euclidean_clusters_fwd': (C.c_int, [VP, VP, VP, C.c_int, C.c_int, C.c_float, C.c_float, C.c_int, C.c_int, VP, VP, VP, VP,
                                                VP]),
    'pvraft_euclidean_clusters_workspace_bytes': (C.c_int64, [C.c_int, C.c_int]),
    'pvraft_rigid_objects_fwd': (C.c_int, [VP, VP, VP, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, C.c_int, C.c_int, VP, VP, VP, VP,
                                           VP, VP, VP, VP, VP, VP, VP]),
    'pvraft_rigid_objects_workspace_bytes': (C.c_int64, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    'pvraft_rigid_objects_fwd_det_workspace_bytes': (C.c_int64, [C.c_int, C.c_int, C.c_int]),
    'pvraft_rigid_objects_bwd': (C.c_int, [VP, VP, VP, VP, VP, VP, VP, C.c_int, C.c_int, C.c_int, VP, VP, VP]),
    'pvraft_sizeof': (C.c_int, [C.c_int]),
    'pvraft_transpose_fwd': (C.c_int, [VP, C.c_int, C.c_int, C.c_int, VP, VP]),
}
EXPORTS = tuple(_SIGNATURES)

_lib = None
_lock = threading.Lock()


class PvraftError(RuntimeError):
    pass


def lib():
    """The loaded shared library (built on first use if nvcc is available; otherwise an error)."""
    global _lib
    if _lib is None:
        with _lock:
            if _lib is None:
                if not os.path.exists(LIB_PATH):
                    from . import build as _build
                    try:
                        _build.build()
                    except Exception as e:   # noqa: BLE001
                        raise PvraftError(f'libpvraft_b200.so is missing and could not be built: {e}') from e
                handle = C.CDLL(LIB_PATH)
                for name, (res, args) in _SIGNATURES.items():
                    fn = getattr(handle, name)    # AttributeError => header/library mismatch: fail loudly
                    fn.restype = res
                    fn.argtypes = args
                _lib = handle
    return _lib


def check(rc, what):
    if rc != 0:
        msg = lib().pvraft_last_error_string()
        raise PvraftError(f'{what} failed (code {rc}): {msg.decode() if msg else "?"}')
