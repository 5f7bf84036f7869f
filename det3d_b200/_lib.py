"""ctypes binding of the det3d_b200 C ABI (include/det3d_b200.h).

The library is the product: there is no Python/CPU fallback.  If the shared
object is missing or a call fails, an exception is raised.
"""
import contextlib
import ctypes as C
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("D3B_LIB") or os.path.join(_HERE, "lib", "libdet3d_b200.so")   # D3B_LIB: development builds

D3B_OK = 0
ALGO_SIMT = 0
ALGO_TC = 1
AA_IOU3D, AA_PIXEL = 0, 1
BOX_XYXYR = 0
BOX_XYWLR = 1
BOX_XYWLR_RRPN = 2
IOU_BEV_XYXYR, OVERLAP_BEV_XYXYR, IOU_BEV_XYWLR = 0, 1, 2     # d3b_boxes_iou_bev modes


class D3BError(RuntimeError):
    pass


class VoxelCfg(C.Structure):
    _fields_ = [
        ("voxel_size", C.c_float * 3),
        ("range_min", C.c_float * 3),
        ("grid", C.c_int32 * 3),
        ("ndim", C.c_int32),
        ("max_points", C.c_int32),
        ("max_voxels", C.c_int32),
    ]


class SiteIndex(C.Structure):
    _fields_ = [
        ("spatial", C.c_int32 * 3),
        ("batch", C.c_int32),
        ("hash_keys", C.c_void_p),
        ("hash_vals", C.c_void_p),
        ("hash_cap", C.c_int32),
        ("bitmap", C.c_void_p),
        ("word_prefix", C.c_void_p),
        ("n_words", C.c_int64),
    ]


class ConvParams(C.Structure):
    _fields_ = [
        ("c_in", C.c_int32),
        ("c_out", C.c_int32),
        ("k_vol", C.c_int32),
        ("weight", C.c_void_p),
        ("weight_packed", C.c_void_p),
        ("bias", C.c_void_p),
        ("scale", C.c_void_p),
        ("shift", C.c_void_p),
        ("residual", C.c_void_p),
        ("relu", C.c_int32),
        ("algo", C.c_int32),
    ]


class Conv16Params(C.Structure):
    _fields_ = [
        ("c_in", C.c_int32), ("c_out", C.c_int32), ("k_vol", C.c_int32),
        ("in_hi", C.c_void_p), ("in_lo", C.c_void_p), ("in_f32", C.c_void_p),
        ("weight", C.c_void_p), ("weight_packed", C.c_void_p), ("acc_scale", C.c_float),
        ("bias", C.c_void_p), ("scale", C.c_void_p), ("shift", C.c_void_p),
        ("residual_hi", C.c_void_p), ("residual_lo", C.c_void_p), ("relu", C.c_int32),
        ("out_hi", C.c_void_p), ("out_lo", C.c_void_p), ("out_f32", C.c_void_p), ("overflow", C.c_void_p),
        ("in_f32_ld", C.c_int32),
    ]


class Bev16Params(C.Structure):
    _fields_ = [
        ("batch", C.c_int32), ("h_in", C.c_int32), ("w_in", C.c_int32), ("c_in", C.c_int32),
        ("c_out", C.c_int32), ("ksize", C.c_int32), ("stride", C.c_int32), ("pad", C.c_int32),
        ("groups", C.c_int32), ("cgroups", C.c_int32), ("up", C.c_int32),
        ("in_hi", C.c_void_p), ("in_lo", C.c_void_p), ("weight_packed", C.c_void_p), ("acc_scale", C.c_float),
        ("bias", C.c_void_p), ("scale", C.c_void_p), ("shift", C.c_void_p), ("relu", C.c_int32),
        ("out_channels", C.c_int32), ("out_c0", C.c_int32),
        ("out_hi", C.c_void_p), ("out_lo", C.c_void_p), ("out_f32", C.c_void_p), ("overflow", C.c_void_p),
    ]


class PredictParams(C.Structure):
    _fields_ = [
        ("cls", C.c_void_p), ("cls_row_stride", C.c_int32), ("cls_col0", C.c_int32),
        ("box", C.c_void_p), ("box_row_stride", C.c_int32), ("box_col0", C.c_int32),
        ("dir", C.c_void_p), ("dir_row_stride", C.c_int32), ("dir_col0", C.c_int32),
        ("anchors", C.c_void_p),
        ("batch", C.c_int32), ("hw", C.c_int32), ("na", C.c_int32), ("n_cls", C.c_int32), ("code", C.c_int32),
        ("nd", C.c_int32),
        ("vec_encode", C.c_int32), ("smooth_dim", C.c_int32), ("norm_velo", C.c_int32),
        ("use_rotate_nms", C.c_int32), ("pre_max", C.c_int32), ("post_max", C.c_int32),
        ("nms_iou_threshold", C.c_float), ("score_threshold", C.c_float), ("direction_offset", C.c_float),
        ("post_center_range", C.c_float * 6), ("has_range", C.c_int32),
        ("label_offset", C.c_int32),
    ]


_I3 = C.c_int32 * 3
_vp, _i32, _i64, _sz, _f32 = C.c_void_p, C.c_int32, C.c_int64, C.c_size_t, C.c_float

# name -> (restype, argtypes); mirrors include/det3d_b200.h one to one.
SIGNATURES = {
    "d3b_last_error": (C.c_char_p, []),
    "d3b_abi_version": (C.c_int, []),
    "d3b_launch_count": (C.c_ulonglong, []),
    "d3b_set_pdl": (None, [C.c_int]),
    "d3b_set_bev_variant": (None, [C.c_int]),
    "d3b_get_bev_variant": (C.c_int, []),
    "d3b_voxelize_workspace_bytes": (_sz, [C.POINTER(VoxelCfg), _i32, _i32]),
    "d3b_voxelize": (C.c_int, [C.POINTER(VoxelCfg), _vp, C.POINTER(_i32), _i32, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "d3b_voxelize_dev": (C.c_int, [C.POINTER(VoxelCfg), _vp, _i32, _vp, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "d3b_ingest_workspace_bytes": (_sz, [_i32]),
    "d3b_ingest_sweeps": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _f32, _vp, _i32, _vp, _vp, _sz, _vp]),
    "d3b_ingest_dev_workspace_bytes": (_sz, [_i32, _i32]),
    "d3b_ingest_sweeps_dev": (C.c_int, [_vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _f32, _vp, _vp, _vp, _vp, _sz, _vp]),
    "d3b_ingest_gather_workspace_bytes": (_sz, [_i32, _i32]),
    "d3b_ingest_sweeps_gather": (C.c_int, [_vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _f32, _vp, _vp, _vp, _vp, _sz, _vp]),
    "d3b_frustum_crop_workspace_bytes": (_sz, [_i32, _i32]),
    "d3b_frustum_crop_dev": (C.c_int, [_vp, _i32, _i32, _vp, _vp, _i32, _vp, _vp, _vp, _vp, _sz, _vp]),
    "d3b_kitti_results_dev": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _vp, _vp, _vp]),
    "d3b_nusc_results_dev": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _vp, _vp, _vp]),
    "d3b_rulebook_workspace_bytes": (_sz, [_i64]),
    "d3b_index_build_hash": (C.c_int, [_vp, _vp, _i32, C.POINTER(SiteIndex), _vp]),
    "d3b_rulebook_subm": (C.c_int, [_vp, _vp, _i32, C.POINTER(SiteIndex), _I3, _vp, _vp, _vp]),
    "d3b_rulebook_conv": (C.c_int, [_vp, _vp, _i32, C.POINTER(SiteIndex), _I3, _I3, _I3, C.POINTER(SiteIndex), _vp, _vp, _i32, _vp, _vp, _vp, _sz, _vp]),
    "d3b_conv_packed_weight_floats": (_sz, [_i32, _i32, _i32]),
    "d3b_conv_pack_weight": (C.c_int, [_vp, _i32, _i32, _i32, _vp, _vp]),
    "d3b_sparse_conv": (C.c_int, [_vp, _vp, _vp, _vp, _i32, C.POINTER(ConvParams), _vp, _vp]),
    "d3b_sparse_to_dense": (C.c_int, [_vp, _vp, _vp, _i32, _i32, _I3, _i32, _vp, _vp]),
    "d3b_pillar_features": (C.c_int, [_vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp, _vp, C.c_float, C.c_float, C.c_float, C.c_float, _vp, _vp]),
    "d3b_voxelize_point_lists": (_vp, [C.POINTER(VoxelCfg), _i32, _i32, _vp]),
    "d3b_pillar_features_lists": (C.c_int, [_vp, _vp, _vp, _i32, _i32, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp, _vp, C.c_float, C.c_float, C.c_float, C.c_float, _vp, _vp]),
    "d3b_sparse_to_bev_rows": (C.c_int, [_vp, _vp, _vp, _i32, _i32, _I3, _i32, _vp, _vp]),
    "d3b_rulebook_dense2d": (C.c_int, [_i32, _i32, _i32, C.c_int32 * 2, C.c_int32 * 2, _vp, _vp, _vp, _vp]),
    "d3b_conv16_packed_weight_halves": (_sz, [_i32, _i32, _i32]),
    "d3b_conv16_pack_weight": (C.c_int, [_vp, _i32, _i32, _i32, _i32, _vp, _vp]),
    "d3b_sparse_conv16": (C.c_int, [_vp, _vp, _vp, _i32, C.POINTER(Conv16Params), _vp]),
    "d3b_split16": (C.c_int, [_vp, _i64, _vp, _vp, _vp, _vp]),
    "d3b_merge16": (C.c_int, [_vp, _vp, _i64, _vp, _vp]),
    "d3b_sparse_to_bev16": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _i32, _i32, _I3, _i32, _vp, _vp, _vp, _vp]),
    "d3b_bev_conv16": (C.c_int, [C.POINTER(Bev16Params), _vp]),
    "d3b_bev_conv16_chain_workspace_bytes": (_i64, [_i32, _i32, _i32, _i32]),
    "d3b_bev_conv16_chain": (C.c_int, [C.POINTER(Bev16Params), _i32, _vp, _i64, _vp]),
    "d3b_predict_workspace_bytes": (_sz, [C.POINTER(PredictParams)]),
    "d3b_predict_task": (C.c_int, [C.POINTER(PredictParams), _vp, _i32, _i32, _vp, _vp, _sz, _vp]),
    "d3b_boxes_iou_bev": (C.c_int, [_vp, _i32, _vp, _i32, _i32, _vp, _vp]),
    "d3b_rotate_iou_rrpn": (C.c_int, [_vp, _i32, _vp, _i32, _i32, _vp, _vp]),
    "d3b_nms_workspace_bytes": (_sz, [_i32]),
    "d3b_rotate_nms": (C.c_int, [_vp, _i32, _vp, _i32, _f32, _i32, _vp, _vp, _vp, _sz, _vp]),
    "d3b_normal_nms": (C.c_int, [_vp, _i32, _vp, _i32, _f32, _i32, _vp, _vp, _vp, _sz, _vp]),
}

_lib = None
_lock = threading.Lock()


def lib():
    """Load (once) and return the C-ABI library; raises if it is not built."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is None:
            if not os.path.exists(LIB_PATH):
                raise D3BError(
                    "det3d_b200 native library missing at %s -- run `python -m det3d_b200.build` "
                    "(there is no CPU fallback)" % LIB_PATH
                )
            handle = C.CDLL(LIB_PATH)
            for name, (res, args) in SIGNATURES.items():
                fn = getattr(handle, name)
                fn.restype = res
                fn.argtypes = args
            _lib = handle
    return _lib


def check(status, what=""):
    if status != D3B_OK:
        msg = lib().d3b_last_error()
        raise D3BError("%s failed (status %d): %s" % (what or "det3d_b200 call", status, (msg or b"").decode()))


def ptr(t):
    """Device (or host) pointer of a torch tensor / None."""
    return None if t is None else t.data_ptr()


def current_stream():
    import torch

    return torch.cuda.current_stream().cuda_stream


@contextlib.contextmanager
def on_device_of(*tensors):
    """Scope a group of C-ABI calls to the device that owns `tensors`.

    The kernels launch on `current_stream()`, i.e. on the CURRENT device's stream, so that device must be the one
    the pointers live on.  All tensors must share one device; when it already is the current one (the usual case:
    one process per GPU) this costs one integer compare."""
    import torch

    dev = None
    for t in tensors:
        if t is None or not torch.is_tensor(t) or not t.is_cuda:
            continue
        if dev is None:
            dev = t.device
        elif t.device != dev:
            raise D3BError("det3d_b200: tensors of one call live on different devices (%s vs %s)" % (dev, t.device))
    if dev is None or dev.index is None or dev.index == torch.cuda.current_device():
        yield
    else:
        with torch.cuda.device(dev):
            yield


# bench.py hook: when set to a list, `timed(tag)` brackets the enclosed C-ABI calls with CUDA events recorded on the
# launching (current) stream and appends (tag, start, end, info) -- per-stage kernel times for the roofline entries.
PROFILE_EVENTS = None


# bench.py hook, in-graph stage times: when set to a list and the current stream is being CAPTURED, `timed(tag)` records one
# external timing event (an event-record node of the graph, cudaEventRecordExternal) whenever the stage tag changes on the
# capture's origin stream -- a handful of nodes at stage boundaries, none between the launches of a stage (those keep their
# programmatic edges).  After a replay, consecutive marks give each stage's duration inside the graph.
GRAPH_MARKS = None


def graph_mark(tag):
    marks = GRAPH_MARKS
    if marks is None:
        return
    import torch

    if not torch.cuda.is_current_stream_capturing():
        return
    st = torch.cuda.current_stream()
    if marks and (marks[0][2] != st.cuda_stream or marks[-1][0] == tag):
        return          # a side stream of the capture (rulebook chain, forked task chains), or still the same stage
    ev = torch.cuda.Event(enable_timing=True, external=True)
    ev.record(st)
    marks.append((tag, ev, st.cuda_stream))


@contextlib.contextmanager
def timed(tag, **info):
    if GRAPH_MARKS is not None:
        graph_mark(tag)
    events = PROFILE_EVENTS
    if events is None:
        yield
        return
    import torch

    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    try:
        yield
    finally:
        ev1.record()
        events.append((tag, ev0, ev1, info))


def launch_count():
    return int(lib().d3b_launch_count())
