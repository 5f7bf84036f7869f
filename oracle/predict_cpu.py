"""TEST INFRASTRUCTURE -- CPU restatement of MultiGroupHead.predict for any Det3D head config.

Follows det3d/models/bbox_heads/mg_head.py:697-1085 (predict / get_task_detections,
use_multi_class_nms=False branch), det3d/core/bbox/box_torch_ops.py:80-148 (second_box_decode,
7- and 9-dim boxes, optional angle-vector encoding), :220-281,349-407 (center_to_corner_box2d,
corner_to_standup_nd), :506-549 (nms -> oracle.aa_nms.nms_pixel, rotate_nms ->
oracle.second_cpu.rotate_nms -> the C restatement of rotate_nms_cc).
"""
import numpy as np
import torch

from .aa_nms import nms_pixel
from .second_cpu import rotate_nms, rotate_nms_cc


def second_box_decode(enc, anchors, encode_angle_to_vector=False, smooth_dim=False, norm_velo=False):
    nd = anchors.shape[-1]
    if nd == 9:
        xa, ya, za, wa, la, ha, vxa, vya, ra = torch.split(anchors, 1, dim=-1)
        if encode_angle_to_vector:
            xt, yt, zt, wt, lt, ht, vxt, vyt, rtx, rty = torch.split(enc, 1, dim=-1)
        else:
            xt, yt, zt, wt, lt, ht, vxt, vyt, rt = torch.split(enc, 1, dim=-1)
    else:
        xa, ya, za, wa, la, ha, ra = torch.split(anchors, 1, dim=-1)
        if encode_angle_to_vector:
            xt, yt, zt, wt, lt, ht, rtx, rty = torch.split(enc, 1, dim=-1)
        else:
            xt, yt, zt, wt, lt, ht, rt = torch.split(enc, 1, dim=-1)
    diagonal = torch.sqrt(la ** 2 + wa ** 2)
    ret = [xt * diagonal + xa, yt * diagonal + ya, zt * ha + za]
    if smooth_dim:
        ret += [(wt + 1) * wa, (lt + 1) * la, (ht + 1) * ha]
    else:
        ret += [torch.exp(wt) * wa, torch.exp(lt) * la, torch.exp(ht) * ha]
    if encode_angle_to_vector:
        rg = torch.atan2(rty + torch.sin(ra), rtx + torch.cos(ra))
    else:
        rg = rt + ra
    if nd > 7:
        ret += [vxt * diagonal + vxa, vyt * diagonal + vya] if norm_velo else [vxt + vxa, vyt + vya]
    ret.append(rg)
    return torch.cat(ret, dim=-1)


def predict_sample_task(cls_logits, box_enc, dir_logits, anchors, test_cfg, vec_encode, direction_offset=0.0):
    """One sample, one task (CPU tensors) -> (boxes [K,nd], scores [K], labels [K])."""
    nd = anchors.shape[-1]
    box_preds = second_box_decode(box_enc.float(), anchors.float(), vec_encode)
    total = torch.sigmoid(cls_logits.float())
    if total.shape[-1] == 1:
        top_scores, top_labels = total.squeeze(-1), torch.zeros(total.shape[0], dtype=torch.long)
    else:
        top_scores, top_labels = torch.max(total, dim=-1)
    thr = test_cfg["score_threshold"]
    keep = top_scores >= thr
    top_scores = top_scores[keep]
    if top_scores.shape[0] == 0:
        return torch.zeros((0, nd)), torch.zeros(0), torch.zeros(0, dtype=torch.long)
    box_preds, top_labels = box_preds[keep], top_labels[keep]
    dir_labels = torch.max(dir_logits, dim=-1)[1][keep] if dir_logits is not None else None
    nms = test_cfg["nms"]
    sel = rotate_nms(box_preds[:, [0, 1, 3, 4, nd - 1]], top_scores, nms["nms_pre_max_size"], nms["nms_post_max_size"],
                     nms["nms_iou_threshold"])
    bx, sc, lb = box_preds[sel].clone(), top_scores[sel], top_labels[sel]
    if dir_labels is not None and bx.shape[0]:
        opp = ((bx[..., -1] - direction_offset) > 0) ^ dir_labels[sel].bool()
        bx[..., -1] += torch.where(opp, torch.tensor(np.pi).type_as(bx), torch.tensor(0.0).type_as(bx))
    rng = torch.tensor(test_cfg["post_center_limit_range"], dtype=torch.float32)
    if bx.shape[0]:
        m = (bx[:, :3] >= rng[:3]).all(1) & (bx[:, :3] <= rng[3:]).all(1)
        bx, sc, lb = bx[m], sc[m], lb[m]
    return bx, sc, lb


def center_to_corner_box2d(centers, dims, angles):
    """box_torch_ops.py:220-255 (corners_nd, origin 0.5: x0y0, x0y1, x1y1, x1y0) and :349-362,388-407 (rotation_2d:
    x' = x cos + y sin, y' = -x sin + y cos, then the centre added).  [N,2], [N,2], [N] -> [N,4,2]."""
    norm = torch.tensor([[0.0, 0.0], [0.0, 1.0], [1.0, 1.0], [1.0, 0.0]], dtype=dims.dtype) - 0.5
    corners = dims.view(-1, 1, 2) * norm.view(1, 4, 2)
    s, c = torch.sin(angles), torch.cos(angles)
    rot_mat_t = torch.stack([torch.stack([c, -s]), torch.stack([s, c])])          # [2,2,N]
    corners = torch.einsum("aij,jka->aik", corners, rot_mat_t)
    return corners + centers.view(-1, 1, 2)


def corner_to_standup_nd(corners):
    """box_torch_ops.py:274-281: [N,4,2] -> [N,4] = min x, min y, max x, max y."""
    return torch.cat([corners.min(dim=1)[0], corners.max(dim=1)[0]], dim=1)


def predict_task_reference(cls_logits, box_enc, dir_logits, anchors, score_threshold, pre_max, post_max,
                           iou_threshold, use_rotate_nms=True, center_range=None, direction_offset=0.0,
                           vec_encode=False, smooth_dim=False, norm_velo=False):
    """get_task_detections (mg_head.py:984-1085, use_multi_class_nms=False) for one sample and one task, on CPU.

    cls_logits [A,C], box_enc [A,code], dir_logits [A,2] | None, anchors [A,nd]; center_range: 6 floats or None.
    Returns a dict of numpy arrays:
      anchor   [K]      anchor index of every box NMS kept, in output order (after post_max)
      boxes    [K,nd]   fp32 boxes, direction flip applied
      boxes64  [K,nd]   the same boxes decoded and flipped in float64 from the same fp32 inputs
      scores   [K], labels [K]
      valid    [K]      the inclusive post_center_limit_range mask; the reference returns the rows where it holds
      nms_in   [N]      anchor indices entering NMS (the top-pre_max passing anchors, by descending score)
      nms_boxes [N,5]   what NMS compared: [x, y, w, l, r] (rotated) or the standup [x1, y1, x2, y2]
    Order among exactly equal scores is the reference's implementation-defined order; here it is the anchor index."""
    logits = cls_logits.float()
    nd = anchors.shape[-1]
    total = torch.sigmoid(logits)
    if total.shape[-1] == 1:
        top_scores, top_labels = total.squeeze(-1), torch.zeros(total.shape[0], dtype=torch.long)
    else:
        # first maximal SCORE; torch.max propagates NaN (an anchor with any NaN class logit scores NaN)
        top_scores, top_labels = torch.max(total, dim=-1)
        top_scores = torch.where(torch.isnan(logits).any(-1), torch.full_like(top_scores, float("nan")), top_scores)
    idx = torch.arange(logits.shape[0])
    if score_threshold > 0.0:
        keep = top_scores >= torch.tensor([score_threshold], dtype=torch.float32)
        idx = idx[keep]
    s = top_scores[idx].numpy()
    order = np.argsort(-s, kind="stable")[:pre_max]                     # torch.topk(pre_max)
    nms_in = idx.numpy()[order]
    nms_scores = s[order]
    enc_sel, anc_sel = box_enc[nms_in].float(), anchors[nms_in].float()
    boxes = second_box_decode(enc_sel, anc_sel, vec_encode, smooth_dim, norm_velo)
    if nms_in.shape[0] == 0:
        keep = np.zeros(0, np.int64)
        nms_boxes = np.zeros((0, 5), np.float32)
    elif use_rotate_nms:
        nms_boxes = boxes[:, [0, 1, 3, 4, nd - 1]].numpy()
        keep = rotate_nms_cc(np.concatenate([nms_boxes, nms_scores[:, None]], 1), iou_threshold)
    else:
        corners = center_to_corner_box2d(boxes[:, :2], boxes[:, 3:5], boxes[:, nd - 1])
        nms_boxes = corner_to_standup_nd(corners).numpy()
        keep = nms_pixel(np.concatenate([nms_boxes, nms_scores[:, None]], 1), iou_threshold)
    keep = np.asarray(keep, np.int64)[:post_max]
    anchor = nms_in[keep]
    bx = boxes[keep].clone()
    bx64 = second_box_decode(enc_sel[keep].double(), anc_sel[keep].double(), vec_encode, smooth_dim, norm_velo)
    sc = torch.from_numpy(nms_scores[keep])
    lb = top_labels[torch.from_numpy(anchor)]
    if dir_logits is not None and bx.shape[0]:
        dir_labels = torch.max(dir_logits[torch.from_numpy(anchor)], dim=-1)[1]
        opp = ((bx[..., -1] - direction_offset) > 0) ^ dir_labels.bool()
        bx[..., -1] += torch.where(opp, torch.tensor(np.pi).type_as(bx), torch.tensor(0.0).type_as(bx))
        bx64[..., -1] += opp.double() * float(np.float32(np.pi))
    if center_range is not None and bx.shape[0]:
        rng = torch.tensor(center_range, dtype=torch.float32)
        m = ((bx[:, :3] >= rng[:3]).all(1) & (bx[:, :3] <= rng[3:]).all(1)).numpy()
    else:
        m = np.ones(bx.shape[0], bool)
    return dict(anchor=anchor, boxes=bx.numpy(), boxes64=bx64.numpy(), scores=sc.numpy(), labels=lb.numpy(), valid=m,
                nms_in=nms_in, nms_boxes=nms_boxes)
