"""Workspace sizes and refusals of every entry point that takes a caller-provided workspace.

The sizes are pinned as recorded numbers: a workspace layout may be reorganised, but what the size functions report
(and so what callers allocate) must not move without a test change.  The refusal matrix checks, without a device,
that a missing or short workspace is refused before anything reaches CUDA, and that exactly enough passes the check."""
import ctypes
import threading

import pytest

from test_abi import _has_cuda_device

# (arguments, bytes) per size function: sizes computed on the host alone, so they are the same with or without a device
HOST_SIZES = {
    "ba": [((36, 8, 40, 80, 1, 8), 4019712), ((72, 8, 40, 80, 1, 8), 7174144), ((1, 2, 4, 4, 1, 2), 6912),
           ((200, 30, 48, 64, 0, 30), 20556544), ((0, 8, 40, 80, 1, 8), 953856), ((36, 0, 40, 80, 1, 8), 0),
           ((36, 8, 40, 80, 1, 9), 0), ((36, 8, 0, 80, 1, 8), 0)],
    "conv_gru": [((1, 48, 64), 1672960), ((12, 40, 80), 20908288), ((3, 5, 7), 70912), ((0, 48, 64), 256),
                 ((1, 0, 64), 256), ((-1, 4, 4), 256)],
    "update_op": [((12, 5, 40, 80), 160582144), ((12, 0, 40, 80), 139282944), ((1, 1, 8, 8), 333824),
                  ((3, -2, 5, 7), 438784), ((0, 1, 8, 8), 256), ((4, 2, 0, 8), 256)],
    "encoder": [((1, 384, 512, 0), 12582912), ((2, 384, 512, 1), 26353664), ((1, 64, 96, 1), 415744),
                ((3, 8, 8, 0), 12288), ((1, 60, 96, 1), 0), ((1, 64, 96, 7), 0), ((0, 64, 96, 0), 0)],
    "frame_distance_grid": [((0, 10, 0, 10), 512), ((5, 40, 0, 45), 1280), ((0, 1000, 100, 1200), 33792),
                            ((3, 3, 0, 5), 0), ((-1, 4, 0, 4), 0)],
    "mvfilter": [((0, 48, 64), 256), ((8, 48, 64), 49664), ((16, 384, 512), 6291968), ((1, 1, 1), 1024),
                 ((-1, 4, 4), 0), ((65536, 4, 4), 0), ((4, 0, 4), 0)],
    "proximity": [((0, 0, 10), 1792), ((5, 0, 40), 22272), ((3, 7, 20), 3328), ((0, 0, 1), 768), ((10, 0, 10), 0),
                  ((-1, 0, 5), 0)],
    "mapping_snapshot": [((1, 48, 64), 61952), ((6, 16, 24), 46592), ((10, 680, 1200), 163264000), ((0, 16, 24), 0),
                         ((1, 0, 4), 0), ((65536, 4, 4), 0)],
    "mc": [((2, 2, 2), 1280), ((32, 32, 32), 37632), ((256, 256, 256), 19072256), ((33, 17, 9), 6656),
           ((1, 4, 4), 0)],
    "mesh_cull": [((0, 0), 1280), ((1, 0), 1280), ((100, 200), 4608), ((123457, 246913), 4445952), ((-1, 0), 0)],
    "icp": [((1,), 1280), ((1000,), 29184), ((123457,), 3492608), ((0,), 0), ((1 << 29,), 0)],
    "neus": [((1, 8), 4864), ((1 << 18, 72), 4864), ((0, 0), 4864)],
}

# sizes that include CUB's temporary storage, which CUB sizes for the device (recorded on an H100)
DEVICE_SIZES = {
    "mesh_sample": [((1,), 1536), ((200,), 4608), ((123457,), 1977344), ((0,), 0)],
    "nn_index": [((1,), 27904), ((1000,), 78848), ((123457,), 6466304), ((0,), 0)],
    "mesh_components": [((3, 1), 4096), ((100, 200), 26368), ((123457, 246913), 29032704), ((0, 0), 3584),
                        ((-1, 0), 0)],
    "mapping_points": [((1, 48, 64), 4608), ((6, 16, 24), 3840), ((10, 680, 1200), 8671488), ((0, 16, 24), 0)],
    "hull": [((1,), 33024), ((500,), 156160), ((123457,), 30896896), ((0,), 0)],
    "ape": [((0,), 2816), ((1,), 2816), ((64,), 5888), ((123457,), 9577984), ((-1,), 0)],
}


def _size(lib, name, args):
    return getattr(lib, "goslam_%s_workspace_bytes" % name)(*args)


def test_host_sized_workspaces(lib):
    got = {name: [(args, _size(lib, name, args)) for args, _ in cases] for name, cases in HOST_SIZES.items()}
    assert got == HOST_SIZES


@pytest.mark.gpu
def test_device_sized_workspaces(lib):
    got = {name: [(args, _size(lib, name, args)) for args, _ in cases] for name, cases in DEVICE_SIZES.items()}
    assert got == DEVICE_SIZES


P = 1 << 20       # a dummy device pointer: never dereferenced, nothing reaches a device


def _entries(lib):
    """name -> (call(workspace, workspace_bytes), bytes the entry requires, or None where CUB sizes the workspace).
    Every call has valid, non-empty shapes; the CUB-sized ones need a device to size and so are checked only for a
    missing workspace."""
    from goslam_b200 import _lib
    p = P
    peers = _lib.BaPeers(world=1, rank=0, epoch=1)
    peers.system[0] = peers.disps[0] = peers.flags[0] = p
    enc = _lib.EncoderWeights()
    for conv in [enc.stem, enc.out] + [c for blk in enc.block for c in blk]:
        conv.w = conv.b = p
    gru, upd = _lib.GruWeights(), _lib.UpdateWeights()
    neus, neus_out = _lib.NeusParams(p, p, p, p, p), _lib.NeusOut(*[p] * 14)
    one = (ctypes.c_int * 1)(1)                         # host arrays: these arguments are read on the host
    lo, hi = (ctypes.c_float * 3)(-1, -1, -1), (ctypes.c_float * 3)(1, 1, 1)
    # the bundle adjustment, the GRU and the update operator report 256 bytes more than their entry points require
    ba = lib.goslam_ba_workspace_bytes(4, 4, 8, 8, 1, 4) - 256
    ba_shape = (4, 4, 8, 8, 1, 4)
    return {
        "ba": (lambda ws, nb: lib.goslam_ba(p, p, p, p, p, p, None, 0, p, p, *ba_shape, 2, 1e-4, 0.1, 1, None, None,
                                            None, ws, nb, None), ba),
        "ba_phase1": (lambda ws, nb: lib.goslam_ba_phase1(p, p, p, p, p, p, None, 0, p, p, *ba_shape, 1, p, ws, nb,
                                                          None), ba),
        "ba_phase2": (lambda ws, nb: lib.goslam_ba_phase2(p, p, p, *ba_shape, 1e-4, 0.1, 1, 0, 4, p, p, None, ws, nb,
                                                          None), ba),
        "ba_phase1_peers": (lambda ws, nb: lib.goslam_ba_phase1_peers(p, p, p, p, p, None, 0, p, p, *ba_shape, 1,
                                                                      ctypes.byref(peers), ws, nb, None), ba),
        "ba_phase2_peers": (lambda ws, nb: lib.goslam_ba_phase2_peers(p, *ba_shape, 1e-4, 0.1, 1, 0, 4,
                                                                      ctypes.byref(peers), p, p, None, ws, nb, None),
                            ba),
        "conv_gru": (lambda ws, nb: lib.goslam_conv_gru(ctypes.byref(gru), p, p, p, p, p, 2, 8, 16, ws, nb, None),
                     lib.goslam_conv_gru_workspace_bytes(2, 8, 16) - 256),
        "update_op": (lambda ws, nb: lib.goslam_update_op(ctypes.byref(upd), p, p, p, p, p, 3, 2, 8, 16, p, p, p, p, p,
                                                          ws, nb, None),
                      lib.goslam_update_op_workspace_bytes(3, 2, 8, 16) - 256),
        "basic_encoder": (lambda ws, nb: lib.goslam_basic_encoder(ctypes.byref(enc), 1, 128, p, 0, None, None, 1, 32,
                                                                  48, p, None, 0, ws, nb, None),
                          lib.goslam_encoder_workspace_bytes(1, 32, 48, 1)),
        "frame_distance_grid": (lambda ws, nb: lib.goslam_frame_distance_grid(p, p, p, 0, 4, 1, 6, 2, 8, 8, 0.3, p, ws,
                                                                              nb, None),
                                lib.goslam_frame_distance_grid_workspace_bytes(0, 4, 1, 6)),
        "mvfilter_compute": (lambda ws, nb: lib.goslam_mvfilter_compute(p, p, p, p, 0.01, 2, 3, 3, 8, 8, ws, nb, None),
                             lib.goslam_mvfilter_workspace_bytes(3, 8, 8)),
        "mvfilter_commit": (lambda ws, nb: lib.goslam_mvfilter_commit(p, p, ws, nb, 3, 8, 8, p, p, p, p, p, p, p, None),
                            lib.goslam_mvfilter_workspace_bytes(3, 8, 8)),
        "proximity_edges": (lambda ws, nb: lib.goslam_proximity_edges(p, 2, 0, 9, 2, 1, 16.0, 100.0, 0, 0, 64, 0, None,
                                                                      None, 0, p, p, 64, p, ws, nb, None),
                            lib.goslam_proximity_workspace_bytes(2, 0, 9)),
        "mapping_snapshot": (lambda ws, nb: lib.goslam_mapping_snapshot(p, p, p, p, 8, 16, 24, p, p, 2, 0.8, ws, nb, p,
                                                                        None),
                             lib.goslam_mapping_snapshot_workspace_bytes(2, 16, 24)),
        "mapping_rays": (lambda ws, nb: lib.goslam_mapping_rays(ws, nb, 2, 16, 24, p, p, 1, 1, one, one, one, 20.0,
                                                                20.0, 12.0, 8.0, p, p, p, p, 1, None),
                         lib.goslam_mapping_snapshot_workspace_bytes(2, 16, 24)),
        "mc_count": (lambda ws, nb: lib.goslam_mc_count(p, 5, 6, 7, 0.0, ws, nb, p, None),
                     lib.goslam_mc_workspace_bytes(5, 6, 7)),
        "mc_emit": (lambda ws, nb: lib.goslam_mc_emit(p, 5, 6, 7, 0.0, lo, hi, ws, nb, p, 1, p, 1, None),
                    lib.goslam_mc_workspace_bytes(5, 6, 7)),
        "mesh_cull_count": (lambda ws, nb: lib.goslam_mesh_cull_count(p, 30, p, 20, lo, hi, ws, nb, p, None),
                            lib.goslam_mesh_cull_workspace_bytes(30, 20)),
        "mesh_cull_emit": (lambda ws, nb: lib.goslam_mesh_cull_emit(p, 30, p, 20, ws, nb, p, 1, p, 1, None),
                           lib.goslam_mesh_cull_workspace_bytes(30, 20)),
        "mesh_cull_mask_count": (lambda ws, nb: lib.goslam_mesh_cull_mask_count(30, p, 20, p, p, ws, nb, p, None),
                                 lib.goslam_mesh_cull_workspace_bytes(30, 20)),
        "mesh_cull_vertex_ids": (lambda ws, nb: lib.goslam_mesh_cull_vertex_ids(30, 20, ws, nb, p, 1, None),
                                 lib.goslam_mesh_cull_workspace_bytes(30, 20)),
        "neus_forward": (lambda ws, nb: lib.goslam_neus_forward(ctypes.byref(neus), p, p, p, p, 1, 8,
                                                                ctypes.byref(neus_out), ws, nb, None),
                         lib.goslam_neus_workspace_bytes(1, 8)),
        "sample_z": (lambda ws, nb: lib.goslam_sample_z(p, p, p, p, p, None, None, 1, 8, 0, 0, p, p, ws, nb, None),
                     256),
        "mapping_points_count": (lambda ws, nb: lib.goslam_mapping_points_count(p, p, p, p, 3, 8, 8, ws, nb, p, None),
                                 None),
        "mapping_points_emit": (lambda ws, nb: lib.goslam_mapping_points_emit(p, p, p, 3, 8, 8, ws, nb, p, 1, None),
                                None),
        "mesh_sample_surface": (lambda ws, nb: lib.goslam_mesh_sample_surface(p, 30, p, 20, p, 1, p, None, ws, nb,
                                                                              None), None),
        "nn_index_build": (lambda ws, nb: lib.goslam_nn_index_build(p, 30, 0.0, ws, nb, None), None),
        "nn_query": (lambda ws, nb: lib.goslam_nn_query(ws, nb, 30, p, 1, 0.5, p, None, None), None),
        "icp_index": (lambda ws, nb: lib.goslam_icp_point_to_point(p, 20, ws, nb, 30, 0.1, p, 5, 1e-6, 1e-6, p, p,
                                                                   1 << 30, None), None),
        "icp_point_to_point": (lambda ws, nb: lib.goslam_icp_point_to_point(p, 20, p, 1 << 30, 30, 0.1, p, 5, 1e-6,
                                                                            1e-6, p, ws, nb, None), None),
        "mesh_components_count": (lambda ws, nb: lib.goslam_mesh_components_count(p, 30, p, 20, ws, nb, p, None), None),
        "mesh_components_keep": (lambda ws, nb: lib.goslam_mesh_components_keep(20, 3, 0.2, 0, ws, nb, p, None), None),
        "hull_vertices": (lambda ws, nb: lib.goslam_hull_vertices(p, 30, ws, nb, p, None), None),
        "hull_vertices_emit": (lambda ws, nb: lib.goslam_hull_vertices_emit(ws, nb, 30, p, 1, None), None),
        "obb_from_hull": (lambda ws, nb: lib.goslam_obb_from_hull(p, 30, ws, nb, 0.1, p, None), None),
        "ape_sim3": (lambda ws, nb: lib.goslam_ape_sim3(p, p, 16, ws, nb, p, p, None), None),
    }


def _in_fresh_thread(fn):
    out = []
    t = threading.Thread(target=lambda: out.append(fn()))
    t.start()
    t.join()
    return out[0]


@pytest.mark.skipif(_has_cuda_device(), reason="passes dummy device pointers: checked only without a CUDA device")
def test_workspace_refusals(lib):
    entries = _entries(lib)
    # icp_index is goslam_icp_point_to_point's nearest-neighbour index argument, checked like a workspace
    assert len(entries) == 34 + 1
    got, want = {}, {}
    for name, (call, need) in entries.items():
        cases = [(None, need or 1 << 30, -3)]
        if need is not None:
            assert need > 0, name
            cases += [(P, need - 1, -3), (P, need, -2)]
        for ws, nb, rc in cases:
            got[name, ws, nb] = _in_fresh_thread(lambda: call(ws, nb))
            want[name, ws, nb] = rc
    assert got == want
