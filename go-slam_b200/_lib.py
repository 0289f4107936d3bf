"""ctypes binding of libgoslam_b200.so (C-ABI in include/goslam_b200.h).

No CPU fallback lives here or anywhere else in the product path: if the shared library is
missing it is built with nvcc (go-slam_b200/build.py); if a kernel cannot launch the caller
gets a RuntimeError.
"""
import ctypes
import os
import threading

from . import build as _build

_lock = threading.Lock()
_LIB = None

c_void_p, c_int, c_float, c_size_t, c_int64 = (
    ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_size_t, ctypes.c_int64)


class NeusParams(ctypes.Structure):
    _fields_ = [
        ("grid", c_void_p), ("sdf_w", c_void_p), ("sdf_b", c_void_p), ("color_B", c_void_p),
        ("mlp_w", c_void_p), ("bound", c_float * 6), ("rt_bound", c_float * 6),
        ("inv_s", c_float), ("cos_anneal_ratio", c_float),
    ]


class NeusOut(ctypes.Structure):
    _fields_ = [
        ("color", c_void_p), ("depth", c_void_p), ("depth_variance", c_void_p),
        ("normal", c_void_p), ("weight_sum", c_void_p), ("sdf", c_void_p), ("z_mid", c_void_p),
        ("gradient_error", c_void_p), ("alpha", c_void_p), ("grad", c_void_p), ("pos", c_void_p),
        ("rgb", c_void_p), ("mlp_in", c_void_p), ("enc", c_void_p), ("fallback", c_void_p),
    ]


class NeusMlpBwdOut(ctypes.Structure):
    _fields_ = [(n, c_void_p) for n in ("H1", "H2", "dH1", "dH2", "dY8", "dE", "d_out", "h", "pts_hl", "d_grad_total")]


class BaPeers(ctypes.Structure):
    _fields_ = [("world", c_int), ("rank", c_int), ("system", c_void_p * 8), ("disps", c_void_p * 8), ("flags", c_void_p * 8),
                ("epoch", ctypes.c_uint), ("timeout", c_void_p)]


class GruWeights(ctypes.Structure):
    _fields_ = [(n, c_void_p) for n in ("w_zr", "w_q", "w_w", "b_zr", "b_q", "b_w", "w_glo", "b_glo")]


class UpdateWeights(ctypes.Structure):
    _fields_ = [("gru", GruWeights)] + [(n, c_void_p) for n in (
        "corr0_w", "corr0_b", "corr2_w", "corr2_b", "flow0_w", "flow0_b", "flow2_w", "flow2_b", "hid_w", "hid_b",
        "delta_w", "delta_b", "weight_w", "weight_b", "agg1_w", "agg1_b", "agg2_w", "agg2_b", "eta_w", "eta_b",
        "upmask_w", "upmask_b")]


class ConvDesc(ctypes.Structure):
    _fields_ = [("inp", c_void_p * 4), ("cin", c_int * 4), ("cin_off", c_int * 4), ("cin_stride", c_int * 4), ("n_in", c_int),
                ("weight", c_void_p), ("bias", c_void_p), ("taps", c_int), ("cout", c_int), ("cout_pad", c_int), ("act", c_int),
                ("out_scale", c_float), ("out", c_void_p), ("out_f32", c_int), ("out_stride", c_int), ("out_offset", c_int),
                ("split", c_int), ("act2", c_int), ("out2", c_void_p)]


class EncoderConv(ctypes.Structure):
    _fields_ = [("w", c_void_p), ("b", c_void_p)]


class EncoderWeights(ctypes.Structure):
    _fields_ = [("stem", EncoderConv), ("block", (EncoderConv * 3) * 6), ("out", EncoderConv)]


# name -> (restype, argtypes); every symbol include/goslam_b200.h declares
SIGNATURES = {
    "goslam_version": (c_int, []),
    "goslam_sm_arch": (c_int, []),
    "goslam_strerror": (ctypes.c_char_p, [c_int]),
    "goslam_last_cuda_error": (ctypes.c_char_p, []),
    "goslam_corr_index_forward": (c_int, [c_void_p, c_int, c_void_p, c_void_p] + [c_int] * 6 + [c_void_p]),
    "goslam_corr_pyramid_lookup": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p] + [c_int] * 6 + [c_void_p]),
    "goslam_corr_build": (c_int, [c_void_p, c_void_p, c_int, c_void_p] + [c_int] * 5 + [c_void_p]),
    "goslam_fmaps_to_kmajor": (c_int, [c_void_p, c_void_p] + [c_int] * 4 + [c_void_p]),
    "goslam_corr_level_plane_elems": (c_size_t, [c_int] * 4),
    "goslam_corr_pool_build": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p] + [c_int] * 5 + [c_void_p]),
    "goslam_corr_pool_lookup": (c_int, [c_void_p, c_int, c_int, c_void_p, c_int, c_int, c_void_p, c_void_p] + [c_int] * 6 + [c_void_p]),
    "goslam_altcorr_forward": (c_int, [c_void_p] * 4 + [c_int] * 8 + [c_void_p]),
    "goslam_altcorr_pyramid": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p] + [c_int] * 5 + [c_void_p]),
    "goslam_frame_distance": (c_int, [c_void_p] * 6 + [c_int] * 3 + [c_float, c_void_p]),
    "goslam_frame_distance_bidir": (c_int, [c_void_p] * 6 + [c_int] * 3 + [c_float, c_void_p]),
    "goslam_frame_distance_grid_workspace_bytes": (c_size_t, [c_int] * 4),
    "goslam_frame_distance_grid": (c_int, [c_void_p] * 3 + [c_int] * 7 + [c_float, c_void_p, c_void_p, c_size_t,
                                                                        c_void_p]),
    "goslam_projmap": (c_int, [c_void_p] * 7 + [c_int] * 3 + [c_void_p]),
    "goslam_iproj": (c_int, [c_void_p] * 4 + [c_int] * 3 + [c_void_p]),
    "goslam_depth_filter": (c_int, [c_void_p] * 6 + [c_int] * 4 + [c_void_p]),
    "goslam_mvfilter_workspace_bytes": (c_size_t, [c_int] * 3),
    "goslam_mvfilter_compute": (c_int, [c_void_p] * 4 + [c_float, c_int, c_int] + [c_int] * 3 +
                                [c_void_p, c_size_t, c_void_p]),
    "goslam_mvfilter_commit": (c_int, [c_void_p] * 3 + [c_size_t] + [c_int] * 3 + [c_void_p] * 8),
    "goslam_reproject": (c_int, [c_void_p] * 7 + [c_int] * 3 + [c_void_p]),
    "goslam_reproject_motion": (c_int, [c_void_p] * 9 + [c_int] * 3 + [c_void_p]),
    "goslam_ba_workspace_bytes": (c_size_t, [c_int] * 6),
    "goslam_ba": (c_int, [c_void_p] * 7 + [c_int] + [c_void_p] * 2 + [c_int] * 7 +
                  [c_float, c_float, c_int] + [c_void_p] * 3 + [c_void_p, c_size_t, c_void_p]),
    "goslam_ba_system_doubles": (c_size_t, [c_int, c_int]),
    "goslam_ba_phase1": (c_int, [c_void_p] * 7 + [c_int] + [c_void_p] * 2 + [c_int] * 7 +
                         [c_void_p, c_void_p, c_size_t, c_void_p]),
    "goslam_ba_phase2": (c_int, [c_void_p] * 3 + [c_int] * 6 + [c_float, c_float] + [c_int] * 3 +
                         [c_void_p] * 3 + [c_void_p, c_size_t, c_void_p]),
    "goslam_ba_phase1_peers": (c_int, [c_void_p] * 6 + [c_int] + [c_void_p] * 2 + [c_int] * 7 +
                               [ctypes.POINTER(BaPeers), c_void_p, c_size_t, c_void_p]),
    "goslam_ba_phase2_peers": (c_int, [c_void_p] + [c_int] * 6 + [c_float, c_float] + [c_int] * 3 +
                               [ctypes.POINTER(BaPeers)] + [c_void_p] * 4 + [c_size_t, c_void_p]),
    "goslam_ba_peers_wait": (c_int, [ctypes.POINTER(BaPeers), c_void_p]),
    "goslam_peer_alloc": (c_int, [c_size_t, c_void_p, c_void_p]),
    "goslam_peer_free": (c_int, [c_void_p]),
    "goslam_ipc_open": (c_int, [c_void_p, c_void_p]),
    "goslam_ipc_close": (c_int, [c_void_p]),
    "goslam_neus_workspace_bytes": (c_size_t, [c_int, c_int]),
    "goslam_neus_forward": (c_int, [ctypes.POINTER(NeusParams)] + [c_void_p] * 4 + [c_int, c_int] +
                            [ctypes.POINTER(NeusOut), c_void_p, c_size_t, c_void_p]),
    "goslam_neus_composite_backward": (c_int, [ctypes.POINTER(NeusParams)] + [c_void_p] * 13 + [c_int64, c_int64, c_int, c_int] +
                                       [c_void_p] * 5),
    "goslam_neus_grid_backward": (c_int, [ctypes.POINTER(NeusParams)] + [c_void_p] * 5 + [c_int64, c_int, c_int] + [c_void_p] * 6),
    "goslam_neus_mlp_backward": (c_int, [ctypes.POINTER(NeusParams)] + [c_void_p] * 10 + [c_int, c_int] +
                                 [ctypes.POINTER(NeusMlpBwdOut), c_void_p]),
    "goslam_hashgrid_layout": (c_int64, [c_void_p, c_void_p, c_void_p]),
    "goslam_neus_sdf_grid": (c_int, [ctypes.POINTER(NeusParams)] + [c_void_p] * 3 + [c_int] * 3 + [c_void_p, c_void_p]),
    "goslam_mc_workspace_bytes": (c_size_t, [c_int] * 3),
    "goslam_mc_count": (c_int, [c_void_p] + [c_int] * 3 + [ctypes.c_double, c_void_p, c_size_t, c_void_p, c_void_p]),
    "goslam_mc_emit": (c_int, [c_void_p] + [c_int] * 3 + [ctypes.c_double] + [c_void_p] * 3 + [c_size_t] +
                       [c_void_p, c_int64, c_void_p, c_int64, c_void_p]),
    "goslam_mesh_cull_workspace_bytes": (c_size_t, [c_int64, c_int64]),
    "goslam_mesh_cull_count": (c_int, [c_void_p, c_int64, c_void_p, c_int64] + [c_void_p] * 3 + [c_size_t, c_void_p, c_void_p]),
    "goslam_mesh_cull_emit": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_size_t, c_void_p, c_int64, c_void_p,
                                      c_int64, c_void_p]),
    "goslam_neus_vertex_color": (c_int, [ctypes.POINTER(NeusParams), c_void_p, c_int64, c_void_p, c_void_p]),
    "goslam_mesh_cull_mask_count": (c_int, [c_int64, c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p,
                                            c_void_p]),
    "goslam_mesh_cull_vertex_ids": (c_int, [c_int64, c_int64, c_void_p, c_size_t, c_void_p, c_int64, c_void_p]),
    "goslam_mesh_depth_render": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_void_p] + [c_int] * 3 +
                                 [ctypes.c_double] * 6 + [c_void_p, c_void_p]),
    "goslam_mesh_view_masks": (c_int, [c_void_p, c_int64, c_void_p, c_void_p] + [c_int] * 3 + [c_float] * 6 +
                               [c_void_p] * 3),
    "goslam_mesh_components_workspace_bytes": (c_size_t, [c_int64, c_int64]),
    "goslam_mesh_components_count": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_size_t, c_void_p, c_void_p]),
    "goslam_mesh_components_keep": (c_int, [c_int64, c_int64, ctypes.c_double, c_int, c_void_p, c_size_t, c_void_p,
                                            c_void_p]),
    "goslam_sample_z": (c_int, [c_void_p] * 7 + [c_int] * 4 + [c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "goslam_cvx_upsample": (c_int, [c_void_p, c_void_p, c_int, c_void_p] + [c_int] * 4 + [c_void_p]),
    "goslam_proximity_workspace_bytes": (c_size_t, [c_int] * 3),
    "goslam_proximity_edges": (c_int, [c_void_p] + [c_int] * 5 + [c_float, c_float, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                                               c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p,
                                                               c_size_t, c_void_p]),
    "goslam_conv_gru_workspace_bytes": (c_size_t, [c_int] * 3),
    "goslam_conv_gru": (c_int, [ctypes.POINTER(GruWeights)] + [c_void_p] * 5 + [c_int] * 3 + [c_void_p, c_size_t, c_void_p]),
    "goslam_nchw_to_nhwc_f16": (c_int, [c_void_p, c_void_p] + [c_int] * 3 + [c_void_p]),
    "goslam_nhwc_to_nchw_f16": (c_int, [c_void_p, c_void_p] + [c_int] * 3 + [c_void_p]),
    "goslam_nchw_to_nhwc_f16_pad": (c_int, [c_void_p, c_void_p] + [c_int] * 4 + [c_void_p]),
    "goslam_conv2d_nhwc": (c_int, [ctypes.POINTER(ConvDesc)] + [c_int] * 3 + [c_void_p]),
    "goslam_update_op_workspace_bytes": (c_size_t, [c_int] * 4),
    "goslam_update_op": (c_int, [ctypes.POINTER(UpdateWeights)] + [c_void_p] * 5 + [c_int] * 4 + [c_void_p] * 5 +
                         [c_void_p, c_size_t, c_void_p]),
    "goslam_mapping_snapshot_workspace_bytes": (c_size_t, [c_int] * 3),
    "goslam_mapping_snapshot": (c_int, [c_void_p] * 4 + [c_int] * 3 + [c_void_p, c_void_p, c_int, c_float, c_void_p,
                                                                        c_size_t, c_void_p, c_void_p]),
    "goslam_mapping_rays": (c_int, [c_void_p, c_size_t] + [c_int] * 3 + [c_void_p, c_void_p, c_int64, c_int] +
                            [c_void_p] * 3 + [ctypes.c_double] * 4 + [c_void_p] * 4 + [c_int64, c_void_p]),
    "goslam_mapping_all_rays": (c_int, [c_void_p, c_int, c_int] + [ctypes.c_double] * 4 + [c_void_p] * 3),
    "goslam_encoder_workspace_bytes": (c_size_t, [c_int] * 4),
    "goslam_basic_encoder": (c_int, [ctypes.POINTER(EncoderWeights), c_int, c_int, c_void_p, c_int, c_void_p, c_void_p] +
                             [c_int] * 3 + [c_void_p, c_void_p, c_int, c_void_p, c_size_t, c_void_p]),
    "goslam_fill_interpolate": (c_int, [c_void_p] * 5 + [c_int, c_int] + [c_void_p] * 3 + [c_int, c_int] +
                                [c_void_p] * 3),
    "goslam_mesh_sample_workspace_bytes": (c_size_t, [c_int64]),
    "goslam_mesh_sample_surface": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_void_p,
                                           c_void_p, c_size_t, c_void_p]),
    "goslam_nn_index_workspace_bytes": (c_size_t, [c_int64]),
    "goslam_nn_index_build": (c_int, [c_void_p, c_int64, ctypes.c_double, c_void_p, c_size_t, c_void_p]),
    "goslam_nn_query": (c_int, [c_void_p, c_size_t, c_int64, c_void_p, c_int64, ctypes.c_double, c_void_p, c_void_p,
                                c_void_p]),
    "goslam_nn_distance_stats": (c_int, [c_void_p, c_int64, ctypes.c_double, c_void_p, c_void_p]),
    "goslam_icp_workspace_bytes": (c_size_t, [c_int64]),
    "goslam_icp_point_to_point": (c_int, [c_void_p, c_int64, c_void_p, c_size_t, c_int64, ctypes.c_double, c_void_p, c_int,
                                          ctypes.c_double, ctypes.c_double, c_void_p, c_void_p, c_size_t, c_void_p]),
    "goslam_mapping_points_workspace_bytes": (c_size_t, [c_int] * 3),
    "goslam_mapping_points_count": (c_int, [c_void_p] * 4 + [c_int] * 3 + [c_void_p, c_size_t, c_void_p, c_void_p]),
    "goslam_mapping_points_emit": (c_int, [c_void_p] * 3 + [c_int] * 3 + [c_void_p, c_size_t, c_void_p, c_int64,
                                                                          c_void_p]),
    "goslam_hull_workspace_bytes": (c_size_t, [c_int64]),
    "goslam_hull_vertices": (c_int, [c_void_p, c_int64, c_void_p, c_size_t, c_void_p, c_void_p]),
    "goslam_hull_vertices_emit": (c_int, [c_void_p, c_size_t, c_int64, c_void_p, c_int64, c_void_p]),
    "goslam_obb_from_hull": (c_int, [c_void_p, c_int64, c_void_p, c_size_t, ctypes.c_double, c_void_p, c_void_p]),
    "goslam_obb_in_bound": (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_void_p]),
    "goslam_ape_workspace_bytes": (c_size_t, [c_int64]),
    "goslam_ape_sim3": (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_size_t, c_void_p, c_void_p, c_void_p]),
    "goslam_corr_index_backward": (c_int, []),
    "goslam_altcorr_backward": (c_int, []),
}


def lib_path():
    return _build.LIB


def load(build_if_missing=True):
    """Return the loaded CDLL (building it first if the .so is absent)."""
    global _LIB
    with _lock:
        if _LIB is not None:
            return _LIB
        path = lib_path()
        if not os.path.exists(path):
            if not build_if_missing:
                raise RuntimeError("libgoslam_b200.so not built (run python -m __graft_entry__ or "
                                   "go-slam_b200/build.py)")
            _build.build()
        lib = ctypes.CDLL(path)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)          # AttributeError => header/library mismatch
            fn.restype = res
            fn.argtypes = args
        _LIB = lib
        return lib


def check(rc, what):
    if rc != 0:
        msg = load().goslam_strerror(int(rc))
        detail = load().goslam_last_cuda_error() if int(rc) == -2 else b""
        raise RuntimeError("%s failed: %s (code %d)%s" % (what, msg.decode() if msg else "?", rc,
                                                          ": " + detail.decode() if detail else ""))


def ptr(t):
    """device pointer of a torch tensor (or None)."""
    return None if t is None else c_void_p(t.data_ptr())


def stream_ptr():
    import torch
    return c_void_p(torch.cuda.current_stream().cuda_stream)
