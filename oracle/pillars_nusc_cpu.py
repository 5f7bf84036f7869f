"""TEST INFRASTRUCTURE -- CPU restatement of the reference's nuScenes PointPillars inference forward
(examples/point_pillars/configs/nusc_all_point_pillars_mghead_syncbn.py):

  reader / scatter  5-feature pillars            oracle/pillars_cpu.pillar_features / pillar_scatter
  neck              RPN[3,5,5], deblocks Conv2d(k = s = 2) / 1x1 / ConvTranspose2d(k = s = 2)
                                                 oracle/pillars_cpu.rpn_forward_multi (necks/rpn.py:67-159)
  heads / predict   six tasks, 9-dim boxes with angle-vector encoding
                                                 oracle/cbgs_cpu.CbgsCPU.heads / predict_tasks
Never imported by det3d_b200."""
import time

import torch

from .cbgs_cpu import CbgsCPU
from .pillars_cpu import PillarsCPU, rpn_forward_multi


class PillarsNuscCPU(PillarsCPU, CbgsCPU):
    """Pillar backbone of PillarsCPU, multi-task heads and predict of CbgsCPU."""

    @torch.no_grad()
    def forward(self, clouds, stages=None):
        t0 = time.perf_counter()
        voxels, coors, nums = self.voxelize(clouds)
        t1 = time.perf_counter()
        feats, canvas = self.backbone(voxels, coors, nums, len(clouds))
        t2 = time.perf_counter()
        x = rpn_forward_multi(self.sd, canvas, self.cfg.model["neck"])
        heads = self.heads(x)
        t3 = time.perf_counter()
        dets = self.predict_tasks(heads)
        t4 = time.perf_counter()
        self.timings = dict(voxelize=t1 - t0, backbone=t2 - t1, rpn_head=t3 - t2, predict=t4 - t3)
        if stages is not None:
            stages.update(dict(voxels=voxels, coors=coors, nums=nums, pillar_feats=feats, dense=canvas, rpn=x,
                               heads=heads))
        return dets
