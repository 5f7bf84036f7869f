"""TEST INFRASTRUCTURE -- the CPU oracles of oracle/second_cpu.py and oracle/cbgs_cpu.py generalised to the two stock
configs that have more than their tasks / features:

* SecondTasksCPU: SECOND with several single-class tasks (kitti_all: Car, Pedestrian, Cyclist).  Each task's heads
  (mg_head.py:198-230) and predict (mg_head.py:697-1085) as SecondCPU does for task 0, the detections concatenated in
  task order with task t's labels offset by the class count of the tasks before it (mg_head.py:1077-1083).
* CbgsTasksCPU: CBGS on Lyft -- 3 of the 4 point columns into the reader (SecondCPU.backbone already takes the first
  num_input_features), the 2016 x 2016 grid, 7-dim boxes without angle-vector encoding, five tasks, and the direction
  classifier's direction_offset (0.785; mg_head.py:1044-1051), which CbgsCPU does not pass on.

On the configs the original oracles cover, both give their outputs bit for bit (tests/test_stock_configs_more.py).
"""
import time

import torch

from oracle.cbgs_cpu import CbgsCPU
from oracle.predict_cpu import predict_sample_task
from oracle.second_cpu import SecondCPU, rpn_forward, second_box_decode, rotate_nms

import numpy as np
import torch.nn.functional as F


def _direction_offset(cfg):
    head = cfg.model["bbox_head"]
    # mg_head.py: the offset is only used by a head with a direction classifier (loss_aux)
    return float(head.get("direction_offset", 0.0)) if head.get("loss_aux") else 0.0


class SecondTasksCPU(SecondCPU):
    def task_head(self, x, t):
        p = "bbox_head.tasks.%d." % t
        sd = self.sd
        return tuple(F.conv2d(x, sd[p + k + ".weight"], sd[p + k + ".bias"]).permute(0, 2, 3, 1).contiguous()
                     for k in ("conv_box", "conv_cls", "conv_dir"))

    def task_predict(self, box, cls, dirs, t):
        """SecondCPU.predict on task t's anchors (single class per task, direction flip with the head's offset)."""
        tc = self.cfg.test_cfg
        offset = _direction_offset(self.cfg)
        B = box.shape[0]
        anchors = self.anchors[t].unsqueeze(0).expand(B, -1, -1)
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
                opp = ((bx[..., -1] - offset) > 0) ^ dl.bool()
                bx[..., -1] += torch.where(opp, torch.tensor(np.pi).type_as(bx), torch.tensor(0.0).type_as(bx))
                m = (bx[:, :3] >= rng[:3]).all(1) & (bx[:, :3] <= rng[3:]).all(1)
                bx, sc = bx[m], sc[m]
            out.append((bx, sc))
        return out

    def predict_tasks(self, heads):
        per_task = [self.task_predict(box, cls, dirs, t) for t, (box, cls, dirs) in enumerate(heads)]
        res = []
        for b in range(heads[0][0].shape[0]):
            boxes = [d[b][0] for d in per_task]
            res.append(dict(box3d_lidar=torch.cat(boxes), scores=torch.cat([d[b][1] for d in per_task]),
                            label_preds=torch.cat([torch.full((bx.shape[0],), t, dtype=torch.long)
                                                   for t, bx in enumerate(boxes)])))
        return res

    @torch.no_grad()
    def forward(self, clouds, stages=None):
        t0 = time.perf_counter()
        voxels, coors, nums = self.voxelize(clouds)
        t1 = time.perf_counter()
        dense = self.backbone(voxels, coors, nums, len(clouds))
        t2 = time.perf_counter()
        x = rpn_forward(self.sd, dense, self.layer_num)
        heads = [self.task_head(x, t) for t in range(len(self.anchors))]
        t3 = time.perf_counter()
        dets = self.predict_tasks(heads)
        t4 = time.perf_counter()
        self.timings = dict(voxelize=t1 - t0, backbone=t2 - t1, rpn_head=t3 - t2, predict=t4 - t3)
        if stages is not None:
            stages.update(dict(voxels=voxels, coors=coors, nums=nums, dense=dense, rpn=x,
                               heads=[dict(box=h[0], cls=h[1], dir=h[2]) for h in heads]))
        return dets


class CbgsTasksCPU(CbgsCPU):
    def predict_tasks(self, heads):
        tc = self.cfg.test_cfg
        vec = bool(self.cfg.box_coder.get("encode_angle_vector", False)) if hasattr(self.cfg, "box_coder") else True
        offset = _direction_offset(self.cfg)
        B = heads[0]["cls"].shape[0]
        res = []
        for b in range(B):
            boxes, scores, labels, flag = [], [], [], 0
            for t, h in enumerate(heads):
                anchors = self.anchors[t]
                a = anchors.shape[0]
                n_cls = h["cls"][b].numel() // a
                code = h["box"][b].numel() // a
                dirs = h["dir"][b].reshape(a, 2) if "dir" in h else None
                bx, sc, lb = predict_sample_task(h["cls"][b].reshape(a, n_cls), h["box"][b].reshape(a, code), dirs,
                                                 anchors, tc, vec, direction_offset=offset)
                boxes.append(bx); scores.append(sc); labels.append(lb + flag)
                flag += n_cls
            res.append(dict(box3d_lidar=torch.cat(boxes), scores=torch.cat(scores), label_preds=torch.cat(labels)))
        return res
