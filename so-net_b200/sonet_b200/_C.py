"""ctypes binding of libsonet_b200.so (the C-ABI declared in include/sonet_b200.h).

The library is the product: if it is missing, importing any op raises — there is NO Python/CPU
fallback for the CUDA entry points. Tensors cross the boundary as raw device pointers; outputs
are allocated by the caller (here, by the thin wrappers in ops.py with torch.empty).
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(os.path.dirname(_HERE), "lib", "libsonet_b200.so")

_lib = None

c_int = ctypes.c_int
c_void_p = ctypes.c_void_p

# name -> argtypes (restype is always int unless listed in _RESTYPE)
_SIGNATURES = {
    "sonet_index_max_f32": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                            c_void_p],
    "sonet_index_max_cpu_f32": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int],
    "sonet_som_assign": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                         c_void_p, c_void_p, c_void_p, c_void_p],
    "sonet_som_query_topk": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                             c_void_p, c_void_p, c_void_p],
    "sonet_som_mask": [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p],
    "sonet_upconv_im2col_f32": [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p],
    "sonet_pointwise_tc_pack_groups": [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p],
    "sonet_pointwise_tc_grouped_forward": [c_void_p, c_int, c_int, c_int, c_void_p,
                                           ctypes.c_longlong, ctypes.c_float, c_void_p, c_int, c_int,
                                           c_int, c_int, c_int, c_int, c_int, ctypes.c_longlong,
                                           c_void_p, c_void_p, c_void_p],
    "sonet_upconv_hshift_f32": [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p],
    "sonet_bn_partial_slots": [c_int, c_int],
    "sonet_bn_train_forward_f32": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, ctypes.c_float,
                                   c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p],
    "sonet_bn_train_backward_f32": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                                    c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                    c_void_p],
    "sonet_index_max_backward_f32": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p,
                                     c_void_p],
    "sonet_instance_norm_f32": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, ctypes.c_float,
                                c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p],
    "sonet_pointwise_tc_pack_device": [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                       c_void_p],
    "sonet_pointwise_tc_forward_dev": [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                       c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p],
    "sonet_absmax_scale_f32": [c_void_p, ctypes.c_longlong, c_void_p, c_void_p, c_void_p],
    "sonet_wgrad_kpad": [c_int, c_int, c_int],
    "sonet_wgrad_blob_bytes": [c_int, ctypes.c_longlong],
    "sonet_wgrad_small_floats": [c_int],
    "sonet_wgrad_tc_f32": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                           c_void_p, c_void_p, c_void_p, c_void_p],
    "sonet_upconv_fold_weights_f32": [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p],
    "sonet_upconv_dgrad_im2col_f32": [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p],
    "sonet_pointwise_tc_pack_groups_device": [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p,
                                              c_void_p, c_void_p],
    "sonet_pointwise_tc_grouped_forward_dev": [c_void_p, c_int, c_int, c_int, c_void_p,
                                               ctypes.c_longlong, c_void_p, c_void_p, c_int, c_int,
                                               c_int, c_int, c_int, c_int, c_int, ctypes.c_longlong,
                                               c_void_p, c_void_p, c_void_p],
    "sonet_comm_nccl_version": [],
    "sonet_comm_unique_id": [c_void_p],
    "sonet_comm_init": [c_void_p, c_int, c_int, c_void_p],
    "sonet_allgather": [c_void_p, c_void_p, c_void_p, ctypes.c_longlong, c_void_p],
    "sonet_comm_destroy": [c_void_p],
    "sonet_som_train": [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                        c_void_p, c_void_p, c_void_p],
    "sonet_augment_f32": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p,
                          c_void_p, c_void_p, ctypes.c_double, ctypes.c_double, ctypes.c_double,
                          ctypes.c_double, ctypes.c_double, ctypes.c_double, c_void_p, c_void_p,
                          c_void_p, ctypes.c_ulonglong, c_void_p, c_void_p, c_void_p, c_void_p],
    "sonet_sample_points_f32": [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_int,
                                c_int, c_void_p, ctypes.c_ulonglong, c_void_p, c_void_p, c_void_p,
                                c_void_p],
    "sonet_som_decenter": [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                           c_void_p, c_void_p, c_void_p],
    "sonet_pointwise_layer_f32": [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_void_p,
                                  c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_int,
                                  c_void_p, c_void_p],
    "sonet_linear_f32": [c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int,
                         c_void_p, c_void_p],
    "sonet_rowmax_f32": [c_void_p, c_int, c_int, c_void_p, c_void_p],
    "sonet_knn_gather_f32": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p,
                             c_void_p],
    "sonet_knn_assemble_f32": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                               c_int, c_void_p, c_void_p, c_void_p],
    "sonet_node_knn": [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p],
    "sonet_gather_points_f32": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p,
                                c_void_p],
    "sonet_kcopy_mean_f32": [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p],
    "sonet_seg_loss_scratch_bytes": [c_int, c_int],
    "sonet_seg_loss_f32": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                           c_void_p],
    "sonet_seg_iou_f32": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p,
                          c_int, c_void_p, c_void_p, c_void_p, c_void_p],
    "sonet_seg_iou_cpu_f32": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p,
                              c_int, c_void_p, c_void_p, c_void_p, c_int],
    "sonet_retrieval_scratch_bytes": [c_int, c_int, c_int, c_int],
    "sonet_retrieval_rank_f32": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p,
                                 ctypes.c_longlong, c_void_p, c_void_p, c_void_p, c_void_p,
                                 c_void_p],
    "sonet_retrieval_rank_cpu_f32": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p,
                                     c_void_p, c_void_p, c_void_p, c_int],
    "sonet_retrieval_format_cpu": [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p,
                                   c_void_p, c_int],
    "sonet_chamfer_f32": [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                          c_void_p, c_void_p, c_void_p, c_void_p, c_void_p],
    "sonet_pointresnet_tc_blob_bytes": [],
    "sonet_pointresnet_tc_fparam_count": [],
    "sonet_pointresnet_tc_pack": [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                  c_void_p, c_void_p, c_void_p, c_void_p],
    "sonet_pointresnet_tc_forward": [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                     c_void_p],
    "sonet_som_sort_decenter": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                c_int, c_void_p, c_void_p, c_void_p, c_void_p],
    "sonet_pointresnet_tc_pool_forward": [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                          c_void_p, c_int, c_void_p, c_void_p, c_void_p],
    "sonet_som_group_smem_bytes": [c_int, c_int, c_int],
    "sonet_som_group_mode": [c_int, c_int, c_int, c_int, ctypes.c_longlong],
    "sonet_som_group_decenter": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p,
                                 c_void_p, c_void_p, c_void_p, c_void_p, c_void_p],
    "sonet_knn_assemble_pool_f32": [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                    c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p],
    "sonet_pool_keys_init": [c_void_p, ctypes.c_longlong, c_void_p],
    "sonet_pool_finalize": [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p],
    "sonet_pointwise_tc_blob_bytes": [c_int, c_int],
    "sonet_pointwise_tc_pack": [c_void_p, c_int, c_int, c_void_p, c_void_p],
    "sonet_pointwise_tc_forward": [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_void_p,
                                   ctypes.c_float, c_void_p, c_int, c_int, c_void_p, c_void_p,
                                   c_int, c_void_p, c_void_p],
    "sonet_nodegemm_image_bytes": [ctypes.c_longlong, c_int, c_int],
    "sonet_nodegemm_split_pack": [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_void_p,
                                  c_void_p],
    "sonet_nodegemm_tc_forward": [c_void_p, c_int, c_int, c_int, c_void_p, ctypes.c_float, c_void_p,
                                  c_int, c_int, c_int, c_void_p, c_void_p, c_void_p],
    "sonet_knn_mlp_tc_blob_bytes": [],
    "sonet_knn_mlp_tc_pack": [c_void_p, c_void_p, c_void_p],
    "sonet_pointwise_tc_forward_rows": [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_void_p,
                                        ctypes.c_float, c_void_p, c_int, c_int, c_void_p, c_void_p,
                                        c_int, c_void_p, c_void_p],
    "sonet_knn_mlp_tc_forward": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p,
                                 ctypes.c_longlong, ctypes.c_longlong, c_void_p, c_void_p,
                                 ctypes.c_float, c_void_p, c_void_p, c_void_p],
    "sonet_debug_knn_mlp_tc_timeline": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                        c_void_p, ctypes.c_longlong, ctypes.c_longlong, c_void_p,
                                        c_void_p, ctypes.c_float, c_void_p, c_void_p, c_void_p,
                                        c_void_p],
    "sonet_debug_pointresnet_tc_timeline": [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p,
                                            c_void_p, c_void_p, c_void_p],
    "sonet_debug_pointwise_tc_timeline": [c_void_p, c_int, c_int, c_int, c_void_p, ctypes.c_float,
                                          c_int, c_void_p, c_void_p, c_void_p],
    "sonet_debug_tc_mma_rate": [c_int, c_int, c_int, c_int, c_void_p, c_void_p],
    "sonet_debug_pointresnet_tc_pool_timeline": [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p,
                                                 c_void_p, c_void_p, c_int, c_void_p, c_void_p,
                                                 c_void_p, c_void_p],
    "sonet_debug_tc_probe": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p,
                             c_void_p],
    "sonet_last_error_string": [],
    "sonet_version": [],
}
# the opt-in fp16 mode: one entry per eval wgmma entry, same arguments
for _name in ("sonet_pointresnet_tc_forward", "sonet_pointresnet_tc_pool_forward",
              "sonet_pointwise_tc_forward", "sonet_pointwise_tc_forward_rows",
              "sonet_pointwise_tc_grouped_forward", "sonet_knn_mlp_tc_forward"):
    _SIGNATURES[_name + "_f16"] = _SIGNATURES[_name]
F16_ENTRIES = tuple(n for n in _SIGNATURES if n.endswith("_f16"))
# explicit activation code (SONET_ACT_RELU / _ELU) and precision (f16 flag) of the fused kernels
_SIGNATURES["sonet_pointresnet_tc_forward_act"] = [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p,
                                                   c_int, c_int, c_void_p, c_void_p]
_SIGNATURES["sonet_pointresnet_tc_pool_forward_act"] = [c_void_p, c_int, c_int, c_int, c_void_p,
                                                        c_void_p, c_void_p, c_void_p, c_int, c_int,
                                                        c_int, c_void_p, c_void_p, c_void_p]
_SIGNATURES["sonet_knn_mlp_tc_forward_act"] = [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                               c_void_p, ctypes.c_longlong, ctypes.c_longlong,
                                               c_void_p, c_void_p, ctypes.c_float, c_void_p, c_int,
                                               c_int, c_void_p, c_void_p]
ACT_ENTRIES = ("sonet_pointresnet_tc_forward_act", "sonet_pointresnet_tc_pool_forward_act",
               "sonet_knn_mlp_tc_forward_act")
_RESTYPE = {"sonet_last_error_string": ctypes.c_char_p, "sonet_version": ctypes.c_char_p,
            "sonet_pointwise_tc_blob_bytes": ctypes.c_longlong,
            "sonet_knn_mlp_tc_blob_bytes": ctypes.c_longlong,
            "sonet_nodegemm_image_bytes": ctypes.c_longlong,
            "sonet_som_group_smem_bytes": ctypes.c_longlong,
            "sonet_seg_loss_scratch_bytes": ctypes.c_longlong,
            "sonet_retrieval_scratch_bytes": ctypes.c_longlong,
            "sonet_retrieval_format_cpu": ctypes.c_longlong,
            "sonet_wgrad_kpad": ctypes.c_longlong, "sonet_wgrad_blob_bytes": ctypes.c_longlong,
            "sonet_wgrad_small_floats": ctypes.c_longlong}

EXPORTED_SYMBOLS = tuple(_SIGNATURES)


def lib():
    """Load (once) and return the ctypes handle. Raises if the library has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                "libsonet_b200.so not found at %s — build it with `python so-net_b200/build.py` "
                "(there is no fallback path)" % LIB_PATH)
        handle = ctypes.CDLL(LIB_PATH)
        for name, argtypes in _SIGNATURES.items():
            fn = getattr(handle, name)  # AttributeError if a declared symbol is not exported
            fn.argtypes = argtypes
            fn.restype = _RESTYPE.get(name, c_int)
        _lib = handle
    return _lib


def last_error():
    return lib().sonet_last_error_string().decode("utf-8", "replace")


def check(rc, what):
    if rc != 0:
        raise RuntimeError("%s failed (%d): %s" % (what, rc, last_error()))


def ptr(t):
    """Device/host pointer of a tensor as an integer (None -> NULL)."""
    return None if t is None else t.data_ptr()
