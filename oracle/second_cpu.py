"""TEST INFRASTRUCTURE -- CPU restatement of the reference's SECOND inference forward.

Stage by stage, with the reference lines each follows:
  voxelize      oracle/voxel_oracle.c          det3d/ops/point_cloud/point_cloud_ops.py:112-184
  collate       prepend batch index            det3d/torchie/parallel/collate.py:130-137
  reader        per-voxel mean                 det3d/models/readers/voxel_encoder.py:206-211
  backbone      oracle/spconv.py               det3d/models/backbones/scn.py:184-197 (+ external spconv,
                                               PARITY UNPINNED there, see oracle/spconv.py)
  neck          conv/BN/ReLU stack, torch CPU  det3d/models/necks/rpn.py:124-159
  head          1x1 convs, NHWC permute        det3d/models/bbox_heads/mg_head.py:198-230
  predict       decode, sigmoid, score filter, det3d/models/bbox_heads/mg_head.py:697-1085
                top-k, rotate NMS, dir flip,   det3d/core/bbox/box_torch_ops.py:80-148,528-549
                range mask                     det3d/ops/nms/nms_cpu.py:34-45 (oracle/iou3d_oracle.c)
Used by tests/ (end-to-end parity of the CUDA pipeline) and by bench.py's
cpu_baseline / --impl reference legs.  Never imported by det3d_b200.
"""
import ctypes as C
import time

import numpy as np
import torch
import torch.nn.functional as F

from . import build as _build
from . import spconv as ospconv
from . import voxel as ovoxel

_lib = None


def _nms_lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(_build.build())
        _lib.oracle_rotate_nms_cc.restype = C.c_int64
        _lib.oracle_rotate_nms_cc.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_float, C.c_void_p]
    return _lib


def rotate_nms_cc(dets, thresh):
    """dets [N,6] = x,y,w,l,r,score (nms_cpu.py:34-45) -> kept indices (into dets), visiting order."""
    dets = np.ascontiguousarray(dets, np.float32)
    n = dets.shape[0]
    order = np.ascontiguousarray(dets[:, 5].argsort()[::-1].astype(np.int32))
    keep = np.zeros(max(n, 1), np.int64)
    k = _nms_lib().oracle_rotate_nms_cc(dets.ctypes.data, order.ctypes.data, n, float(thresh), keep.ctypes.data)
    return keep[:k]


def rotate_nms(rbboxes, scores, pre_max_size=None, post_max_size=None, iou_threshold=0.5):
    """box_torch_ops.py:528-549 on CPU tensors."""
    indices = None
    if pre_max_size is not None:
        k = min(scores.shape[0], pre_max_size)
        scores, indices = torch.topk(scores, k=k)
        rbboxes = rbboxes[indices]
    dets = torch.cat([rbboxes, scores.unsqueeze(-1)], dim=1).numpy()
    keep = rotate_nms_cc(dets, iou_threshold)[:post_max_size] if len(dets) else np.zeros(0, np.int64)
    keep = torch.from_numpy(np.asarray(keep, np.int64))
    if keep.shape[0] == 0:
        return torch.zeros([0]).long()
    return indices[keep] if indices is not None else keep


def second_box_decode(enc, anchors):
    """box_torch_ops.py:80-148, 7-dim boxes, exp dims, plain angle residual."""
    xa, ya, za, wa, la, ha, ra = torch.split(anchors, 1, dim=-1)
    xt, yt, zt, wt, lt, ht, rt = torch.split(enc, 1, dim=-1)
    diagonal = torch.sqrt(la ** 2 + wa ** 2)
    return torch.cat([xt * diagonal + xa, yt * diagonal + ya, zt * ha + za, torch.exp(wt) * wa,
                      torch.exp(lt) * la, torch.exp(ht) * ha, rt + ra], dim=-1)


def _bn2d(x, sd, prefix, eps=1e-3):
    return F.batch_norm(x, sd[prefix + ".running_mean"], sd[prefix + ".running_var"], sd[prefix + ".weight"],
                        sd[prefix + ".bias"], False, 0.0, eps)


def rpn_forward(sd, x, layer_num):
    """necks/rpn.py:124-159 for the single-block SECOND config (stride 1, 1x1 deblock)."""
    p = "neck.blocks.0."
    x = F.pad(x, (1, 1, 1, 1))
    x = F.relu(_bn2d(F.conv2d(x, sd[p + "1.weight"]), sd, p + "2"))
    idx = 4
    for _ in range(layer_num):
        x = F.relu(_bn2d(F.conv2d(x, sd[p + "%d.weight" % idx], padding=1), sd, p + "%d" % (idx + 1)))
        idx += 3
    d = "neck.deblocks.0."
    return F.relu(_bn2d(F.conv2d(x, sd[d + "0.weight"]), sd, d + "1"))


class SecondCPU:
    """state_dict of the det3d_b200 / Det3D VoxelNet + the config -> CPU forward."""

    def __init__(self, cfg, state_dict, anchors):
        self.cfg = cfg
        self.sd = {k: v.detach().float().cpu() for k, v in state_dict.items() if torch.is_tensor(v)}
        self.anchors = [torch.as_tensor(a).float() for a in anchors]      # per task [A, 7]
        vg = cfg.voxel_generator
        self.vs = np.asarray(vg["voxel_size"], np.float32)
        self.pcr = np.asarray(vg["range"], np.float32)
        self.max_points = vg["max_points_in_voxel"]
        self.max_voxels = vg["max_voxel_num"]
        self.grid = ovoxel.grid_size(self.vs, self.pcr)
        self.arch = cfg.model["backbone"]["type"]
        self.layer_num = cfg.model["neck"]["layer_nums"][0]
        self.timings = {}

    def voxelize(self, clouds):
        vox, coors, nums = [], [], []
        for b, pts in enumerate(clouds):
            v, c, n = ovoxel.points_to_voxel(pts, self.vs, self.pcr, self.max_points, True, self.max_voxels)
            vox.append(v)
            coors.append(np.concatenate([np.full((c.shape[0], 1), b, np.int32), c], 1))
            nums.append(n)
        return np.concatenate(vox), np.concatenate(coors), np.concatenate(nums)

    def backbone(self, voxels, coors, nums, batch, **kw):
        """Reader (per-voxel mean, fp32) + middle encoder; `kw` goes to middle_encoder_forward (dtype, return_levels)."""
        feats = torch.from_numpy(voxels[:, :, : self.cfg.model["reader"]["num_input_features"]]).sum(1) / \
            torch.from_numpy(nums).float().view(-1, 1)
        sd = {k[len("backbone."):]: v for k, v in self.sd.items() if k.startswith("backbone.")}
        return ospconv.middle_encoder_forward(sd, feats, coors, batch, [int(g) for g in self.grid], arch=self.arch, **kw)

    def head(self, x):
        t = "bbox_head.tasks.0."
        sd = self.sd
        box = F.conv2d(x, sd[t + "conv_box.weight"], sd[t + "conv_box.bias"]).permute(0, 2, 3, 1).contiguous()
        cls = F.conv2d(x, sd[t + "conv_cls.weight"], sd[t + "conv_cls.bias"]).permute(0, 2, 3, 1).contiguous()
        dirs = F.conv2d(x, sd[t + "conv_dir.weight"], sd[t + "conv_dir.bias"]).permute(0, 2, 3, 1).contiguous()
        return box, cls, dirs

    def predict(self, box, cls, dirs):
        """mg_head.py:697-1085, single task, use_multi_class_nms=False, sigmoid scores."""
        tc = self.cfg.test_cfg
        B = box.shape[0]
        anchors = self.anchors[0].unsqueeze(0).expand(B, -1, -1)
        reg = second_box_decode(box.view(B, -1, 7), anchors)
        cls = cls.view(B, -1, 1)
        dirs = dirs.view(B, -1, 2)
        rng = torch.tensor(tc["post_center_limit_range"], dtype=torch.float32)
        out = []
        for b in range(B):
            box_preds, dir_labels = reg[b], torch.max(dirs[b], dim=-1)[1]
            top_scores = torch.sigmoid(cls[b]).squeeze(-1)
            keep = top_scores >= tc["score_threshold"]
            top_scores = top_scores[keep]
            if top_scores.shape[0] != 0:
                box_preds, dir_labels = box_preds[keep], dir_labels[keep]
                sel = rotate_nms(box_preds[:, [0, 1, 3, 4, 6]], top_scores, tc["nms"]["nms_pre_max_size"],
                                 tc["nms"]["nms_post_max_size"], tc["nms"]["nms_iou_threshold"])
            else:
                sel = torch.zeros([0]).long()
            bx, sc, dl = box_preds[sel].clone(), top_scores[sel], dir_labels[sel]
            if bx.shape[0]:
                opp = (bx[..., -1] > 0) ^ dl.bool()
                bx[..., -1] += torch.where(opp, torch.tensor(np.pi).type_as(bx), torch.tensor(0.0).type_as(bx))
                m = (bx[:, :3] >= rng[:3]).all(1) & (bx[:, :3] <= rng[3:]).all(1)
                bx, sc = bx[m], sc[m]
            out.append(dict(box3d_lidar=bx, scores=sc, label_preds=torch.zeros(bx.shape[0], dtype=torch.long)))
        return out

    @torch.no_grad()
    def forward(self, clouds, stages=None):
        t0 = time.perf_counter()
        voxels, coors, nums = self.voxelize(clouds)
        t1 = time.perf_counter()
        dense = self.backbone(voxels, coors, nums, len(clouds))
        t2 = time.perf_counter()
        x = rpn_forward(self.sd, dense, self.layer_num)
        box, cls, dirs = self.head(x)
        t3 = time.perf_counter()
        dets = self.predict(box, cls, dirs)
        t4 = time.perf_counter()
        self.timings = dict(voxelize=t1 - t0, backbone=t2 - t1, rpn_head=t3 - t2, predict=t4 - t3)
        if stages is not None:
            stages.update(dict(voxels=voxels, coors=coors, nums=nums, dense=dense, rpn=x, box=box, cls=cls, dirs=dirs))
        return dets
