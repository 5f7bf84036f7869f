"""The C-ABI library must load on a CPU-only host and export every function that
include/det3d_b200.h declares (no compute calls here: there is no GPU)."""
import ctypes
import os
import re

from conftest import ROOT
from det3d_b200 import _lib


def _declared_functions():
    text = open(os.path.join(ROOT, "include", "det3d_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    names = re.findall(r"\b(d3b_[a-z0-9_]+)\s*\(", text)
    return sorted(set(names))


def test_header_functions_are_exported():
    names = _declared_functions()
    assert len(names) >= 15
    handle = ctypes.CDLL(_lib.LIB_PATH)
    missing = [n for n in names if not hasattr(handle, n)]
    assert not missing, "declared in the header but not exported: %s" % missing


def test_binding_table_covers_the_header():
    assert sorted(_lib.SIGNATURES) == _declared_functions()


def _plane_writers():
    """{entry point: (takes out_hi, takes an overflow pointer)} for every function of the header; a parameter counts
    when it is named in the signature or is a field of a params struct the signature takes."""
    text = open(os.path.join(ROOT, "include", "det3d_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    structs = {}
    for body, name in re.findall(r"typedef\s+struct\s*\{(.*?)\}\s*(\w+)\s*;", text, flags=re.S):
        structs[name] = set(re.findall(r"\b(\w+)\s*(?:\[[^\]]*\])?\s*;", body))
    text = re.sub(r"typedef\s+struct\s*\{.*?\}\s*\w+\s*;", "", text, flags=re.S)
    out = {}
    for name, args in re.findall(r"\b(d3b_[a-z0-9_]+)\s*\(([^;{]*?)\)\s*;", text, flags=re.S):
        params = set(re.findall(r"\b(\w+)\s*(?:\[[^\]]*\])?\s*(?:,|$)", args.strip()))
        for t in re.findall(r"\b(\w+)\s*\*", args):
            params |= structs.get(t, set())
        out[name] = ("out_hi" in params, "overflow" in params)
    return out


def test_every_plane_writer_takes_an_overflow_flag():
    """A value that leaves the f16 range cannot be carried by the hi / lo planes, so every entry point that writes planes
    (`out_hi`, as a parameter or a field of its params struct) must take the device flag that reports it."""
    writers = _plane_writers()
    assert len(writers) == len(_declared_functions())
    planes = {n for n, (hi, _) in writers.items() if hi}
    assert {"d3b_sparse_conv16", "d3b_bev_conv16", "d3b_sparse_to_bev16"} <= planes
    missing = sorted(n for n in planes if not writers[n][1])
    assert not missing, "write f16 planes without an overflow flag: %s" % missing


def test_abi_5_and_error_string():
    """ABI 5: the voxelizer and the sweep ingest take their tables from device memory only (d3b_voxelize_dev,
    d3b_ingest_sweeps_dev with a nullable sweep_src); since ABI 4 the rulebook builders take no pair lists."""
    L = _lib.lib()
    assert L.d3b_abi_version() == 5
    assert len(_lib.SIGNATURES["d3b_rulebook_subm"][1]) == 8
    assert len(_lib.SIGNATURES["d3b_rulebook_conv"][1]) == 16
    assert len(_lib.SIGNATURES["d3b_ingest_sweeps_dev"][1]) == 19
    assert isinstance(L.d3b_last_error(), bytes)
    assert L.d3b_launch_count() >= 0


def test_argument_validation_without_gpu():
    # invalid arguments are rejected before any CUDA call is made
    L = _lib.lib()
    assert L.d3b_voxelize_workspace_bytes(None, 10, 1) == 0
    st = L.d3b_sparse_conv(None, None, None, None, 10, None, None, None)
    assert st == 1 and b"null" in L.d3b_last_error()
    cfg = _lib.VoxelCfg()                                   # all zero: no grid, ndim 0
    dummy = (ctypes.c_int32 * 2)()
    st = L.d3b_voxelize_dev(ctypes.byref(cfg), None, 0, dummy, 1, None, dummy, dummy, None, dummy, None, dummy, 0, None)
    assert st == 1 and b"cfg" in L.d3b_last_error()


def test_sparse_conv_rejects_an_unknown_algo_without_gpu():
    """Only D3B_ALGO_SIMT (0) and D3B_ALGO_TC (1) exist: any other value is an invalid argument, never a silent fall
    through to another kernel."""
    L = _lib.lib()
    dummy = (ctypes.c_float * 16)()
    for algo in (2, 3, -1):
        p = _lib.ConvParams(c_in=16, c_out=16, k_vol=27, weight=ctypes.addressof(dummy),
                            weight_packed=ctypes.addressof(dummy), relu=1, algo=algo)
        st = L.d3b_sparse_conv(dummy, dummy, dummy, dummy, 128, ctypes.byref(p), dummy, None)
        assert st == 1 and b"algo" in L.d3b_last_error()


def test_entry_points_validate_before_cuda_without_gpu():
    """Every entry point validates before it touches CUDA: status 1 (invalid argument) / 3 (unsupported) + message."""
    L = _lib.lib()
    i3 = (ctypes.c_int32 * 3)(3, 3, 3)
    assert L.d3b_rulebook_subm(None, None, 10, None, i3, None, None, None) == 1
    assert L.d3b_rulebook_conv(None, None, 10, None, i3, i3, i3, None, None, None, 10, None, None, None, 0, None) == 1
    assert L.d3b_rotate_nms(None, 10, None, 7, 0.5, 10, None, (ctypes.c_int32 * 1)(), None, 0, None) == 1
    assert b"format" in L.d3b_last_error()
    assert L.d3b_normal_nms(None, 10, None, 5, 0.5, 10, None, (ctypes.c_int32 * 1)(), None, 0, None) == 1
    assert b"mode" in L.d3b_last_error()
    # d3b_boxes_iou_bev: modes 0 / 1 (XYXYR IoU / overlap) and 2 (the XYWLR rotate_nms_cc overlap); nothing else
    assert (_lib.IOU_BEV_XYXYR, _lib.OVERLAP_BEV_XYXYR, _lib.IOU_BEV_XYWLR) == (0, 1, 2)
    for mode in (3, -1):
        assert L.d3b_boxes_iou_bev(None, 4, None, 4, mode, None, None) == 1
        assert b"mode" in L.d3b_last_error()
    one = (ctypes.c_float * 8)()
    st = L.d3b_pillar_features(one, one, one, one, 4, 100, 2, 64, one, one, one, 0.16, 0.16, 0.0, 0.0, one, None)
    assert st == 3 and b"ndim" in L.d3b_last_error()                         # D3B_ERR_UNSUPPORTED
    off = (ctypes.c_int32 * 2)(0, 5)
    u8 = (ctypes.c_uint8 * 1)(0)
    lag = (ctypes.c_float * 1)(0.0)
    cloud = (ctypes.c_int32 * 2)()
    # 40 sweeps for one sample, then raw_stride 3 < n_feat 4
    assert L.d3b_ingest_sweeps_dev(None, 5, 5, 4, off, None, off, lag, lag, u8, 40, 1, 1.0, None, cloud, None, cloud,
                                   1 << 20, None) == 1
    assert b"sweep_capacity 40" in L.d3b_last_error()
    assert L.d3b_ingest_sweeps_dev(None, 5, 3, 4, off, None, off, lag, lag, u8, 1, 1, 1.0, None, cloud, None, cloud, 1 << 20,
                                   None) == 1
    assert b"bad layout" in L.d3b_last_error()
    assert L.d3b_ingest_dev_workspace_bytes(-1, 1) == 0 and L.d3b_nms_workspace_bytes(0) == 16
    q = _lib.PredictParams()
    assert L.d3b_predict_workspace_bytes(ctypes.byref(q)) == 0
    assert L.d3b_predict_task(ctypes.byref(q), None, 0, 0, None, None, 0, None) == 1


def test_pillar_reader_rejects_unbuilt_shapes_without_gpu():
    """The pillar reader, both sources: every (ndim, units, max_points, batch) outside what the kernels are built for
    returns its status and a message before any CUDA call -- 3 (unsupported) for ndim / units, 1 (invalid argument)
    for sizes, a list-mode batch above 64, and staging above the 200 KB of shared memory."""
    L = _lib.lib()
    one = (ctypes.c_float * 8)()

    def dense(rows, P, ndim, units):
        return L.d3b_pillar_features(one, one, one, one, rows, P, ndim, units, one, one, one, 0.2, 0.2, 0.1, 0.1, one, None)

    def lists(batch, P, ndim, units):
        return L.d3b_pillar_features_lists(one, one, one, batch, 16, one, one, one, 4, P, ndim, units, one, one, one,
                                           0.2, 0.2, 0.1, 0.1, one, None)

    for call in (dense, lambda *a: lists(2, *a[1:])):
        for ndim, units, status, word in ((12, 64, 3, b"ndim"), (4, 16, 3, b"units"), (4, 48, 3, b"units"),
                                          (5, 160, 3, b"units"), (4, 64, 1, b"bad sizes")):
            st = call(4, 0 if word == b"bad sizes" else 20, ndim, units)
            assert st == status and word in L.d3b_last_error(), (ndim, units, st, L.d3b_last_error())
        # (P, ndim) whose staging (4 warps x P x ndim fp32 + the weights) exceeds 200 KB
        assert ((5 + 5) * 64 + 4 * 2600 * 5) * 4 > 200 * 1024
        assert call(4, 2600, 5, 64) == 1 and b"shared memory" in L.d3b_last_error()
    assert lists(65, 20, 4, 64) == 1 and b"batch 65" in L.d3b_last_error()
    assert lists(0, 20, 4, 64) == 1 and b"batch 0" in L.d3b_last_error()


def test_rulebook_conv_rejects_a_kernel_wider_than_the_padded_input():
    """D = 1, k = 2, padding 0: there is no output cell along z (floor((1 - 2) / 2) + 1 = 0); C's truncating division
    would make it 1, an output whose window leaves the grid.  Rejected before any CUDA call."""
    host = (ctypes.c_int32 * 16)()
    buf = ctypes.addressof(host)
    i3 = lambda *v: (ctypes.c_int32 * 3)(*v)
    in_idx, out_idx = _lib.SiteIndex(), _lib.SiteIndex()
    in_idx.spatial, in_idx.batch = i3(1, 8, 8), 1
    out_idx.spatial, out_idx.batch = i3(1, 4, 4), 1
    out_idx.bitmap, out_idx.word_prefix, out_idx.n_words = buf, buf, 1
    st = _lib.lib().d3b_rulebook_conv(buf, buf, 1, ctypes.byref(in_idx), i3(2, 2, 2), i3(2, 2, 2), i3(0, 0, 0),
                                      ctypes.byref(out_idx), buf, buf, 1, buf, buf, buf, 64, None)
    assert st == 1
    assert b"wider than the padded input" in _lib.lib().d3b_last_error()
