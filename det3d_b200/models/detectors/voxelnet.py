"""VoxelNet single-stage detector (det3d/models/detectors/voxelnet.py:5-52,
single_stage.py:9-36): reader -> sparse middle encoder -> RPN neck -> head."""
import torch
from torch import nn

from .. import builder
from ..registry import DETECTORS


@DETECTORS.register_module
class SingleStageDetector(nn.Module):
    def __init__(self, reader, backbone, neck=None, bbox_head=None, train_cfg=None, test_cfg=None,
                 pretrained=None):
        super().__init__()
        self.reader = builder.build_reader(reader)
        self.backbone = builder.build_backbone(backbone)
        if neck is not None:
            self.neck = builder.build_neck(neck)
        self.bbox_head = builder.build_head(bbox_head)
        self.train_cfg = train_cfg
        self.test_cfg = test_cfg

    @property
    def with_neck(self):
        return hasattr(self, "neck") and self.neck is not None

    def init_weights(self, pretrained=None):
        self.backbone.init_weights(pretrained=pretrained)
        if self.with_neck:
            self.neck.init_weights()
        self.bbox_head.init_weights()


class _FusedBevMixin:
    """Routes RPN + heads through the det3d_b200 tensor-core kernels.

    math = "fp16x3" (default): NHWC split-f16 planes + TMA tensor maps (csrc/bevconv16_sm90.cu), any RPN the
    reference builds; "tf32x3": the round-1 gather kernel (stride-1 RPN only), which is also where a forward is
    re-run when a feature leaves the f16 range (`overflow_flag`)."""
    use_fused_bev = True
    math = "fp16x3"
    _bev16 = None
    _bev32 = None
    _ovf = None

    def set_math(self, math):
        assert math in ("fp16x3", "tf32x3")
        self.math = math
        fused = getattr(self.backbone, "fused", None)
        if fused is not None:
            fused().math = math

    def overflow_flag(self, device):
        if self._ovf is None or self._ovf.device != device:
            self._ovf = torch.zeros(1, dtype=torch.int32, device=device)
        return self._ovf

    def fused_bev(self):
        """The fused (neck, bbox_head) executor for the current math, or None (module forward through torch)."""
        if self.training or not self.with_neck or not self.use_fused_bev:
            return None
        from det3d_b200.ops.spconv import bev
        if self.math == "fp16x3":
            if self._bev16 is None:
                ok = hasattr(self.backbone, "forward_planes") and bev.rpn_is_fusable16(self.neck)
                self._bev16 = bev.FusedBevStack(self.neck, self.bbox_head) if ok else False
            return self._bev16 or None
        if self._bev32 is None:
            ok = hasattr(self.backbone, "forward_rows") and bev.rpn_is_fusable(self.neck)
            self._bev32 = bev.FusedBevStackTF32(self.neck, self.bbox_head) if ok else False
        return self._bev32 or None


@DETECTORS.register_module
class VoxelNet(_FusedBevMixin, SingleStageDetector):

    def extract_feat(self, data):
        feats = self.reader(data["features"], data["num_voxels"])
        x = self.backbone(feats, data["coors"], data["batch_size"], data["input_shape"],
                          **({"n_dev": data["n_dev"]} if data.get("n_dev") is not None else {}))
        return self.neck(x) if self.with_neck else x

    def forward(self, example, return_loss=True, **kwargs):
        num_voxels = example["num_voxels"]
        data = dict(features=example["voxels"], num_voxels=example["num_points"],
                    coors=example["coordinates"], batch_size=len(num_voxels),
                    input_shape=example["shape"][0], n_dev=example.get("n_voxels_dev"))
        bev = self.fused_bev() if not return_loss else None
        if bev is not None and self.math == "fp16x3":
            feats = self.reader(data["features"], data["num_voxels"])
            ovf = self.overflow_flag(feats.device)
            planes = self.backbone.forward_planes(feats, data["coors"], data["batch_size"], data["input_shape"],
                                                  n_dev=data["n_dev"], overflow=ovf)
            preds = bev.run(planes, overflow=ovf)
        elif bev is not None:
            feats = self.reader(data["features"], data["num_voxels"])
            rows, (b, h, w) = self.backbone.forward_rows(feats, data["coors"], data["batch_size"],
                                                          data["input_shape"], n_dev=data["n_dev"])
            preds = bev.run(rows, b, h, w)
        else:
            preds = self.bbox_head(self.extract_feat(data))
        if return_loss:
            return self.bbox_head.loss(example, preds)
        if kwargs.get("device_output", False):
            return self.bbox_head.predict_device(example, preds, self.test_cfg)
        return self.bbox_head.predict(example, preds, self.test_cfg)
