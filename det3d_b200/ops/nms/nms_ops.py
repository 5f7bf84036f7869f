"""Device-side NMS entry points over d3b_rotate_nms / d3b_normal_nms (csrc/nms.cu)."""
import torch

from ... import _lib

_WS = {}


def _workspace(n, device):
    need = _lib.lib().d3b_nms_workspace_bytes(int(n))
    ws = _WS.get(device)
    if ws is None or ws.numel() < need:
        ws = _WS[device] = torch.empty(max(need, 1 << 20), dtype=torch.uint8, device=device)
    return ws


def nms_sorted(boxes_sorted, fmt, thresh, max_keep=None, n_dev=None, axis_aligned=False, out=None,
               aa_mode=_lib.AA_IOU3D):
    """Greedy NMS over boxes already sorted by descending score ([N,5] f32 cuda).

    Returns (keep_idx int64[max_keep], keep_count int32[1]) device tensors -- no host sync.
    """
    assert boxes_sorted.is_cuda and boxes_sorted.dtype == torch.float32 and boxes_sorted.shape[1] == 5
    boxes_sorted = boxes_sorted.contiguous()
    n = boxes_sorted.shape[0]
    max_keep = n if max_keep is None else min(int(max_keep), n)
    dev = boxes_sorted.device
    if out is None:
        keep_idx = torch.empty(max(max_keep, 1), dtype=torch.int64, device=dev)
        keep_count = torch.zeros(1, dtype=torch.int32, device=dev)
    else:
        keep_idx, keep_count = out
    ws = _workspace(n, dev)
    L = _lib.lib()
    with _lib.on_device_of(boxes_sorted, n_dev, keep_idx, keep_count):
        if axis_aligned:
            st = L.d3b_normal_nms(boxes_sorted.data_ptr(), n, _lib.ptr(n_dev), int(aa_mode), float(thresh), max_keep,
                                  keep_idx.data_ptr(), keep_count.data_ptr(), ws.data_ptr(), ws.numel(),
                                  _lib.current_stream())
        else:
            st = L.d3b_rotate_nms(boxes_sorted.data_ptr(), n, _lib.ptr(n_dev), int(fmt), float(thresh), max_keep,
                                  keep_idx.data_ptr(), keep_count.data_ptr(), ws.data_ptr(), ws.numel(),
                                  _lib.current_stream())
    _lib.check(st, "d3b nms")
    return keep_idx, keep_count


def _finish(order, keep_idx, keep_count):
    k = int(keep_count.item())  # API boundary: variable-length result
    return order[keep_idx[:k]]


def rotate_nms_xywlr(rbboxes, scores, iou_threshold, post_max_size=None):
    """[N,5] (x,y,w,l,r) + scores -> kept indices into the input, descending score
    (rotate_nms_cc semantics: `>=`, hull-overlap gate)."""
    order = torch.argsort(scores, descending=True, stable=True)
    keep_idx, keep_count = nms_sorted(rbboxes.float()[order], _lib.BOX_XYWLR, iou_threshold, post_max_size)
    return _finish(order, keep_idx, keep_count)


def normal_nms_xyxy(bboxes, scores, iou_threshold, post_max_size=None, pixel=False):
    """[N,4] (x1,y1,x2,y2) axis-aligned NMS, `>`.  pixel=False: iou3d nms_normal extents;
    pixel=True: the "+1" extents of numba nms_gpu (what box_torch_ops.nms calls, nms_gpu.py:22-33)."""
    order = torch.argsort(scores, descending=True, stable=True)
    b5 = torch.cat([bboxes.float(), bboxes.new_zeros((bboxes.shape[0], 1), dtype=torch.float32)], dim=1)
    keep_idx, keep_count = nms_sorted(b5[order], _lib.BOX_XYXYR, iou_threshold, post_max_size, axis_aligned=True,
                                      aa_mode=_lib.AA_PIXEL if pixel else _lib.AA_IOU3D)
    return _finish(order, keep_idx, keep_count)


def boxes_iou_bev(boxes_a, boxes_b, mode=_lib.IOU_BEV_XYXYR):
    """[na, nb] f32 matrix: mode IOU_BEV_XYXYR / OVERLAP_BEV_XYXYR the iou3d IoU / overlap area of [x1,y1,x2,y2,ry]
    boxes; mode IOU_BEV_XYWLR the rotate_nms_cc overlap of [cx,cy,w,l,r] boxes that BOX_XYWLR NMS thresholds."""
    a = boxes_a.float().contiguous()
    b = boxes_b.float().contiguous()
    out = torch.zeros((a.shape[0], b.shape[0]), dtype=torch.float32, device=a.device)
    with _lib.on_device_of(a, b):
        st = _lib.lib().d3b_boxes_iou_bev(a.data_ptr(), a.shape[0], b.data_ptr(), b.shape[0], int(mode),
                                          out.data_ptr(), _lib.current_stream())
    _lib.check(st, "d3b_boxes_iou_bev")
    return out
