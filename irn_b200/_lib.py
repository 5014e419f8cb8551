"""ctypes binding of libirn_b200.so (the C ABI declared in include/irn_b200.h).

There is NO CPU fallback: if the shared library is missing, or a device entry point is called
without a CUDA device, this raises.  PyTorch is used only for device memory and streams.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("IRN_B200_LIB", os.path.join(_HERE, "libirn_b200.so"))   # override: A/B builds during development

_lib = None

c_int, c_size_t, c_void_p, c_double, c_float = ctypes.c_int, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_double, ctypes.c_float
_p_int = ctypes.POINTER(ctypes.c_int)

# name -> (restype, argtypes); must list every symbol include/irn_b200.h declares
SIGNATURES = {
    "irn_last_error": (ctypes.c_char_p, []),
    "irn_version": (c_int, []),
    "irn_path_index_shape": (c_int, [c_int, _p_int, _p_int, _p_int, _p_int]),
    "irn_path_index_fill": (c_int, [c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "irn_edge_to_affinity": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "irn_to_affinity_forward": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "irn_to_affinity_backward": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "irn_rw_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int, c_int]),
    "irn_random_walk": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_double, c_int,
                                c_void_p, c_size_t, c_void_p]),
    "irn_random_walk_variant": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_double,
                                        c_int, c_void_p, c_size_t, c_int, c_void_p]),
    "irn_rw_last_launch_count": (c_int, []),
    "irn_rw_last_was_fused": (c_int, []),
    "irn_total_launch_count": (ctypes.c_longlong, []),
    "irn_rw_set_timing": (c_int, [c_int]),
    "irn_rw_last_step_ms": (c_int, [ctypes.POINTER(c_float), _p_int]),
    "irn_cam_net_create": (c_int, [c_void_p, c_size_t, ctypes.POINTER(c_void_p)]),
    "irn_irn_net_create": (c_int, [c_void_p, c_size_t, ctypes.POINTER(c_void_p)]),
    "irn_net_destroy": (None, [c_void_p]),
    "irn_net_set_conv_mode": (c_int, [c_void_p, c_int]),
    "irn_net_get_conv_mode": (c_int, [c_void_p]),
    "irn_conv_create": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, ctypes.POINTER(c_void_p)]),
    "irn_conv_destroy": (None, [c_void_p]),
    "irn_conv_forward": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "irn_stem_create": (c_int, [c_void_p, c_void_p, ctypes.POINTER(c_void_p)]),
    "irn_stem_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "irn_stem_forward": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int, c_void_p, c_size_t,
                                 c_void_p]),
    "irn_shortcut_conv_create": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, ctypes.POINTER(c_void_p)]),
    "irn_shortcut_conv_forward": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "irn_cam_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "irn_cam_forward": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
    "irn_edge_displacement_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int]),
    "irn_edge_displacement_forward": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                              c_size_t, c_void_p]),
    "irn_cam_merge": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p,
                              c_void_p]),
    "irn_find_centroids": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "irn_connected_components": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "irn_cluster_scratch_bytes": (c_size_t, [c_int, c_int]),
    "irn_cluster_centroids": (c_int, [c_void_p, c_void_p, c_float, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "irn_instance_seeds": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "irn_segment_stats": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "irn_segment_masks": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "irn_rw_labels": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p, c_void_p, c_void_p,
                              c_void_p, c_void_p, c_void_p]),
    "irn_jpeg_decoder_create": (c_int, [c_int, ctypes.POINTER(c_void_p)]),
    "irn_jpeg_decoder_backend": (c_int, [c_void_p]),
    "irn_jpeg_decoder_destroy": (None, [c_void_p]),
    "irn_jpeg_image_size": (c_int, [c_void_p, c_void_p, c_size_t, _p_int, _p_int, _p_int]),
    "irn_jpeg_decode_batch": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_void_p]),
    "irn_resize_ksize": (c_int, [c_int, c_int]),
    "irn_resize_coeffs": (c_int, [c_int, c_int, c_void_p, c_void_p]),
    "irn_normalize_lut": (c_int, [c_void_p, c_void_p, c_void_p]),
    "irn_resize_plan_create": (c_int, [c_int, c_int, c_int, c_int, c_void_p, c_void_p, ctypes.POINTER(c_void_p)]),
    "irn_resize_plan_destroy": (c_int, [c_void_p]),
    "irn_resize_workspace_bytes": (c_size_t, [c_void_p, c_int]),
    "irn_resize_forward": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "irn_crf_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int, c_int]),
    "irn_crf_max_labels": (c_int, []),
    "irn_dense_crf": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_double, c_float, c_float, c_float, c_float,
                              c_float, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "irn_ir_label": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_float, c_float, c_void_p, c_void_p,
                             c_void_p, c_size_t, c_void_p]),
    "irn_crf_set_timing": (c_int, [c_int]),
    "irn_crf_last_ms": (c_int, [ctypes.POINTER(c_float)]),
}


class IrnError(RuntimeError):
    pass


def lib():
    """Load (once) and return the ctypes handle.  Raises if the library was not built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise IrnError("libirn_b200.so not found at %s -- run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(there is no CPU fallback)" % LIB_PATH)
        h = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(h, name)          # AttributeError if the ABI and the header drifted apart
            fn.restype = res
            fn.argtypes = args
        _lib = h
    return _lib


def check(rc, what=""):
    if rc != 0:
        msg = lib().irn_last_error()
        raise IrnError("%s failed (%d): %s" % (what or "libirn_b200 call", rc, msg.decode() if msg else "?"))


def stream_ptr():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise IrnError("irn_b200 device entry points take CUDA tensors only (no CPU fallback); got %s" % t.device)


def ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)
