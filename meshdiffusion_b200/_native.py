"""ctypes binding of libmeshdiff_b200.so (the C ABI declared in include/meshdiff_b200.h).

There is deliberately no fallback: if the library is missing or a call fails, an exception is raised.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libmeshdiff_b200.so")

_lib = None


class NativeError(RuntimeError):
    pass


class UNetConfigC(ctypes.Structure):
    _fields_ = [
        ("image_size", ctypes.c_int),
        ("nf", ctypes.c_int),
        ("n_levels", ctypes.c_int),
        ("ch_mult", ctypes.c_int * 8),
        ("num_res_blocks", ctypes.c_int),
        ("level0_blocks", ctypes.c_int),
        ("n_attn", ctypes.c_int),
        ("attn_resolutions", ctypes.c_int * 4),
        ("num_channels", ctypes.c_int),
        ("stem_ksize", ctypes.c_int),
        ("use_pos_bias", ctypes.c_int),
        ("max_batch", ctypes.c_int),
        ("precision", ctypes.c_int),
        ("training", ctypes.c_int),
        ("num_classes", ctypes.c_int),
    ]


class SamplerCondC(ctypes.Structure):
    """mdb_sampler_cond (include/meshdiff_b200.h)."""
    _fields_ = [
        ("partial", ctypes.c_void_p), ("partial_bstride", ctypes.c_longlong),
        ("partial_mask", ctypes.c_void_p), ("mask_bstride", ctypes.c_longlong),
        ("channel", ctypes.c_int), ("mean_coef", ctypes.c_float), ("std", ctypes.c_float),
        ("noise", ctypes.c_void_p),
    ]


class DistillRowC(ctypes.Structure):
    """mdb_distill_row (include/meshdiff_b200.h)."""
    _fields_ = [(name, ctypes.c_float) for name in
                ("label_s", "label_m", "label_e", "sigma_s", "inv_alpha_s", "c_x_s", "c_0_s",
                 "sigma_m", "inv_alpha_m", "c_x_m", "c_0_m", "r", "inv_d")]


class SolverEntryC(ctypes.Structure):
    """mdb_solver_entry (include/meshdiff_b200.h)."""
    _fields_ = [("kind", ctypes.c_int)] + [(name, ctypes.c_float) for name in
                                           ("label", "sigma", "inv_alpha", "c_x", "c_0", "c_1", "c_z", "known_coef",
                                            "known_std")]


class SolverKnownC(ctypes.Structure):
    """mdb_solver_known (include/meshdiff_b200.h)."""
    _fields_ = [
        ("known", ctypes.c_void_p), ("known_bstride", ctypes.c_longlong),
        ("mask", ctypes.c_void_p), ("mask_bstride", ctypes.c_longlong),
        ("channels", ctypes.c_uint), ("noise", ctypes.c_void_p),
    ]


class GemmSrcC(ctypes.Structure):
    """mdb_gemm_src (include/meshdiff_b200.h)."""
    _fields_ = [("ptr", ctypes.c_void_p), ("channels", ctypes.c_int), ("x", ctypes.c_int), ("y", ctypes.c_int),
                ("z", ctypes.c_int), ("ld", ctypes.c_longlong)]


PROBE_CONV, PROBE_CONV_UP2, PROBE_CONV_DGRAD, PROBE_POINTWISE, PROBE_ACT_B = range(5)


class GemmProbeDescC(ctypes.Structure):
    """mdb_gemm_probe_desc (include/meshdiff_b200.h)."""
    _fields_ = [
        ("precision", ctypes.c_int), ("kind", ctypes.c_int), ("ksize", ctypes.c_int), ("stride", ctypes.c_int),
        ("parity", ctypes.c_int), ("n_src", ctypes.c_int), ("src", GemmSrcC * 2),
        ("w", ctypes.c_void_p), ("w_in_out", ctypes.c_int),
        ("b_ptr", ctypes.c_void_p), ("b_k", ctypes.c_int), ("b_n", ctypes.c_int),
        ("b_row_stride", ctypes.c_longlong), ("b_batch_stride", ctypes.c_longlong),
        ("n_extra", ctypes.c_int), ("extra", GemmSrcC * 2), ("w_extra", ctypes.c_void_p),
        ("x", ctypes.c_int), ("y", ctypes.c_int), ("z", ctypes.c_int), ("n", ctypes.c_int), ("out", ctypes.c_void_p),
        ("osx", ctypes.c_longlong), ("osy", ctypes.c_longlong), ("osz", ctypes.c_longlong), ("osb", ctypes.c_longlong),
        ("lo_off", ctypes.c_longlong), ("out_fp32", ctypes.c_int),
        ("bias", ctypes.c_void_p), ("rowbias", ctypes.c_void_p), ("rowbias_ld", ctypes.c_longlong),
        ("residual", ctypes.c_void_p), ("res_ld", ctypes.c_longlong), ("res_batch_stride", ctypes.c_longlong),
        ("stats", ctypes.c_void_p), ("alpha", ctypes.c_float), ("splits", ctypes.c_int),
        ("batch_plan", ctypes.c_int), ("batch", ctypes.c_int), ("dry", ctypes.c_int),
        ("gnb", ctypes.c_int), ("gn_x0", ctypes.c_void_p), ("gn_c0", ctypes.c_int), ("gn_x1", ctypes.c_void_p),
        ("gn_c1", ctypes.c_int), ("gn_stats0", ctypes.c_void_p), ("gn_stats1", ctypes.c_void_p),
        ("gn_gamma", ctypes.c_void_p), ("gn_beta", ctypes.c_void_p), ("gn_silu", ctypes.c_int),
        ("gn_dropout", ctypes.c_float), ("gn_seed", ctypes.c_ulonglong),
        ("gn_dx", ctypes.c_void_p), ("gn_dgamma", ctypes.c_void_p), ("gn_dbeta", ctypes.c_void_p),
    ]


class GemmProbeReportC(ctypes.Structure):
    """mdb_gemm_probe_report (include/meshdiff_b200.h)."""
    _fields_ = [("work_items", ctypes.c_int), ("splits", ctypes.c_int), ("ksteps", ctypes.c_int),
                ("entry_ksteps", ctypes.c_int), ("block_n", ctypes.c_int), ("flops", ctypes.c_double),
                ("fill_bytes", ctypes.c_double)]


# name -> (restype, argtypes); the symbol list is checked against the header by tests/test_abi.py
_vp, _i, _ll, _f, _u64, _d = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_float, ctypes.c_ulonglong, ctypes.c_double
SIGNATURES = {
    "mdb_last_error": (ctypes.c_char_p, []),
    "mdb_version": (_i, []),
    "mdb_unet_create": (_i, [ctypes.POINTER(UNetConfigC), ctypes.POINTER(_vp)]),
    "mdb_unet_create_dry": (_i, [ctypes.POINTER(UNetConfigC), ctypes.POINTER(_vp)]),
    "mdb_unet_destroy": (None, [_vp]),
    "mdb_unet_num_params": (_i, [_vp]),
    "mdb_unet_param_info": (_i, [_vp, _i, ctypes.POINTER(ctypes.c_char_p), ctypes.POINTER(_ll), ctypes.POINTER(_i), ctypes.POINTER(_ll)]),
    "mdb_unet_set_param": (_i, [_vp, ctypes.c_char_p, _vp, _ll, _i, _vp]),
    "mdb_unet_get_param": (_i, [_vp, ctypes.c_char_p, _vp, _ll, _i, _vp]),
    "mdb_unet_commit": (_i, [_vp, _vp]),
    "mdb_unet_set_params": (_i, [_vp, _i, _vp, _vp, _vp, _vp]),
    "mdb_unet_forward": (_i, [_vp, _vp, _vp, _vp, _i, _vp]),
    "mdb_unet_info": (_i, [_vp, ctypes.POINTER(_d), ctypes.POINTER(_ll), ctypes.POINTER(_i), ctypes.POINTER(_i)]),
    "mdb_unet_gemm_ops": (_i, [_vp, _i, ctypes.POINTER(ctypes.c_char_p), ctypes.POINTER(_d), ctypes.POINTER(_d)]),
    "mdb_unet_gemm_slots": (_i, [_vp, _i, ctypes.POINTER(_i), ctypes.POINTER(_i), ctypes.POINTER(_i)]),
    "mdb_unet_gemm_tiles": (_i, [_vp, _i, ctypes.POINTER(_i), ctypes.POINTER(_i), ctypes.POINTER(_i), ctypes.POINTER(_i),
                                 ctypes.POINTER(_i)]),
    "mdb_unet_profile": (_i, [_vp, _vp, _vp, _vp, _i, _vp, ctypes.c_char_p, _i, ctypes.POINTER(_f), _i, ctypes.POINTER(_i)]),
    "mdb_unet_set_dropout": (_i, [_vp, _f, _u64]),
    "mdb_unet_set_classes": (_i, [_vp, _vp, _i, _vp]),
    "mdb_unet_backward": (_i, [_vp, _vp, _vp, _ll, _i, _i, _vp]),
    "mdb_unet_grad_offset": (_i, [_vp, ctypes.c_char_p, ctypes.POINTER(_ll)]),
    "mdb_unet_backward_input": (_i, [_vp, _vp, _vp, _vp, _ll, _i, _i, _vp]),
    "mdb_unet_grad_ready": (_i, [_vp, ctypes.c_char_p, ctypes.POINTER(_i)]),
    "mdb_unet_backward_marked": (_i, [_vp, _vp, _vp, _ll, _i, _i, ctypes.POINTER(_i), ctypes.POINTER(_vp), _i, _vp]),
    "mdb_unet_debug_stats": (_i, [_vp, _vp, _ll, ctypes.POINTER(_ll)]),
    "mdb_unet_train_info": (_i, [_vp, ctypes.POINTER(_d), ctypes.POINTER(_i), ctypes.POINTER(_ll)]),
    "mdb_unet_profile_backward": (_i, [_vp, _vp, _vp, _i, _vp, ctypes.c_char_p, _i, ctypes.POINTER(_f), _i, ctypes.POINTER(_i)]),
    "mdb_fingerprint": (_i, [_vp, _vp, _i, _vp, _vp]),
    "mdb_sampler_update": (_i, [_vp, _vp, _vp, _vp, _vp, _f, _f, _ll, _i, _i, _u64, _u64, ctypes.POINTER(SamplerCondC), _vp]),
    "mdb_sampler_run": (_i, [_vp, _vp, _vp, _vp, ctypes.POINTER(_f), ctypes.POINTER(_f), ctypes.POINTER(_f), _i, _i, _u64, _vp, _vp,
                             _i, ctypes.POINTER(SamplerCondC), ctypes.POINTER(_f), ctypes.POINTER(_f), _i, _vp]),
    "mdb_solver_update": (_i, [_vp, _vp, _vp, _vp, ctypes.POINTER(SolverEntryC), _ll, _i, _i, _vp, _u64, _u64,
                               ctypes.POINTER(SolverKnownC), _vp]),
    "mdb_solver_run": (_i, [_vp, _vp, _vp, _vp, ctypes.POINTER(SolverEntryC), _i, _i, _u64, _vp, _vp, _i,
                            ctypes.POINTER(SolverKnownC), _i, _vp]),
    "mdb_solver_update_guided": (_i, [_vp, _vp, _f, _vp, _vp, _vp, ctypes.POINTER(SolverEntryC), _ll, _i, _i, _vp, _u64, _u64,
                                      ctypes.POINTER(SolverKnownC), _vp]),
    "mdb_solver_run_guided": (_i, [_vp, _vp, _vp, _vp, ctypes.POINTER(SolverEntryC), _i, _i, _u64, _vp, _f, _vp, _vp, _vp, _i,
                                   ctypes.POINTER(SolverKnownC), _i, _vp]),
    "mdb_distill_step": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _vp, _ll, _i, _i, _vp]),
    "mdb_distill_targets": (_i, [_vp, _vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp, _i, _vp]),
    "mdb_ddpm_loss": (_i, [_vp, _vp, _vp, _d, _vp, _vp, _vp, _i, _i, _ll, _vp]),
    "mdb_ddpm_perturb": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _ll, _vp]),
    "mdb_chunk_elems": (_i, []),
    "mdb_grad_clip_coef": (_i, [_vp, _vp, _vp, _i, _f, _vp, _vp, _vp, _vp]),
    "mdb_adam_ema_step": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _f, _f, _f, _f, _f, _i, _vp, _f, _vp]),
    "mdb_ema_update": (_i, [_vp, _vp, _vp, _vp, _i, _f, _vp]),
    "mdb_allreduce_grads": (_i, [_vp, _vp, _ll, _i, _vp]),
    "mdb_conv3d": (_i, [_vp, _i, _i, _i, _i, _i, _vp, _vp, _i, _i, _i, _vp, _vp, _vp, _vp, _i, _vp]),
    "mdb_groupnorm_act": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _ll, _i, _i, _i, _vp]),
    "mdb_conv3d_backward": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp]),
    "mdb_groupnorm_act_backward": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _ll, _i, _i, _f, _u64, _vp]),
    "mdb_conv3d_backward_prec": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _i, _vp]),
    "mdb_groupnorm_act_backward_prec": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _ll, _i, _i, _f, _u64, _i, _vp]),
    "mdb_gemm_probe": (_i, [ctypes.POINTER(GemmProbeDescC), ctypes.POINTER(GemmProbeReportC), _vp]),
    "mdb_upsample_conv": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, ctypes.POINTER(GemmProbeReportC), _vp]),
    "mdb_attention_core": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, ctypes.POINTER(GemmProbeReportC), _vp]),
    "mdb_marching_tets_prepare": (_i, [_vp, _i, _i, _i, ctypes.POINTER(_vp)]),
    "mdb_marching_tets_destroy": (None, [_vp]),
    "mdb_marching_tets_info": (_i, [_vp, ctypes.POINTER(_i), ctypes.POINTER(_i)]),
    "mdb_marching_tets_uvs": (_i, [_vp, _vp, _vp]),
    "mdb_marching_tets_count": (_i, [_vp, _vp, _i, ctypes.POINTER(_i), _vp]),
    "mdb_mesh_auto_normals": (_i, [_vp, _vp, _i, _i, _vp, _vp, _vp, _vp]),
    "mdb_mesh_compute_tangents": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _vp, _vp, _vp]),
    "mdb_marching_tets_extract": (_i, [_vp, _vp, _ll, _vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "mdb_marching_tets_vertex_ids": (_i, [_vp, _i, _vp, _vp]),
    "mdb_marching_tets_backward": (_i, [_vp, _vp, _ll, _vp, _i, _vp, _vp, _vp, _vp, _vp, _vp]),
    "mdb_mesh_sample_points": (_i, [_vp, _vp, _vp, _vp, _i, _i, _vp, _u64, _ll, _vp, _vp, _vp, _vp]),
    "mdb_chamfer_matrix": (_i, [_vp, _i, _i, _vp, _i, _i, _vp, _vp]),
    "mdb_chamfer_pairs": (_i, [_vp, _i, _i, _vp, _i, _vp, _vp, _vp, _vp]),
    "mdb_emd_matrix": (_i, [_vp, _i, _vp, _i, _i, _f, _vp, _vp, _vp]),
    "mdb_pflow_drift_div": (_i, [_vp, _vp, _vp, _vp, _vp, _f, _f, _vp, _vp, _i, _i, _ll, _vp]),
    "mdb_raster_depth": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    "mdb_visible_tets": (_i, [_vp, _ll, _vp, _i, _vp, _vp, _vp, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    "mdb_render_shade": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "mdb_carve_vertices": (_i, [_vp, _i, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp]),
    "mdb_closest_points": (_i, [_vp, _vp, _i, _ll, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "mdb_nearest_vertex": (_i, [_vp, _vp, _i, _ll, _vp, _vp, _vp, _vp, _vp]),
    "mdb_segment_sum": (_i, [_vp, _i, _vp, _vp, _ll, _vp, _vp]),
    "mdb_depth_unproject": (_i, [_vp, _i, _i, _vp, _vp, _f, _vp, _vp, _vp, _vp, _vp]),
    "mdb_depth_closest_points": (_i, [_vp, _vp, _i, _ll, _i, _vp, _vp, _f, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "mdb_lfd_descriptors": (_i, [_vp, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    "mdb_lfd_matrix": (_i, [_vp, _i, _vp, _i, _vp, _vp, _vp]),
    "mdb_slerp_chunks": (_i, []),
    "mdb_slerp_frames": (_i, [_vp, _vp, _ll, _i, ctypes.POINTER(_d), _i, _vp, _vp, _vp, _vp, _vp]),
}


def lib():
    """Loads the shared library (building it in-tree first if the sources are newer)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        from . import build as _build
        _build.build()
    if not os.path.exists(LIB_PATH):
        raise NativeError("libmeshdiff_b200.so is missing and could not be built; there is no fallback path")
    L = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(L, name)
        fn.restype = res
        fn.argtypes = args
    _lib = L
    return L


def check(code):
    if code != 0:
        raise NativeError(lib().mdb_last_error().decode())


def ptr(t):
    """Raw device/host pointer of a torch tensor (None -> NULL)."""
    if t is None:
        return None
    return ctypes.c_void_p(t.data_ptr())


def current_stream():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
