"""VoxelNet single-stage detector (det3d/models/detectors/voxelnet.py:5-52,
single_stage.py:9-36): reader -> sparse middle encoder -> RPN neck -> head."""
import torch
from torch import nn

from .. import builder
from ..registry import DETECTORS

MATHS = ("fp16x3", "fp16", "tf32x3")     # convolution arithmetic of the fused path (_FusedBevMixin.set_math)
F16_MATHS = ("fp16x3", "fp16")           # the ones on f16 planes


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
    reference builds; "fp16" (opt-in): the same kernels on the hi plane alone, one MMA per product -- faster, not
    fp32-equivalent (DESIGN 3.0); "tf32x3": the output-stationary 3xTF32 gather kernel over a dense rulebook
    (csrc/sparse_conv_sm90.cu, stride-1 RPN only), which is also where a forward is re-run when a feature leaves the f16
    range (`overflow_flag`)."""
    use_fused_bev = True
    math = "fp16x3"
    fp16_enabled = False        # set by det3d.core.fp16.wrap_fp16_model
    _ovf = None

    def set_math(self, math):
        if math not in MATHS:
            raise ValueError("unknown math %r: one of %s" % (math, ", ".join(MATHS)))
        self.math = math
        fused = getattr(self.backbone, "fused", None)
        if fused is not None:
            fused().math = math

    def n_planes(self):
        """f16 planes per activation on the fused path: 1 for "fp16", 2 for "fp16x3"."""
        return 1 if self.math == "fp16" else 2

    def overflow_flag(self, device):
        # "cuda" (the pipeline's device) and "cuda:0" (a tensor's) must name the same flag: comparing them unresolved
        # swapped in a fresh zero flag on every call, and the host never saw one the kernels had raised
        device = torch.device(device)
        if device.type == "cuda" and device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        if self._ovf is None or self._ovf.device != device:
            self._ovf = torch.zeros(1, dtype=torch.int32, device=device)
        return self._ovf

    def fused_bev(self):
        """The fused (neck, bbox_head) executor for the current math, or None (module forward through torch)."""
        if self.training or not self.with_neck or not self.use_fused_bev:
            return None
        from det3d_b200.ops.spconv import bev
        cache = self.__dict__.setdefault("_fused_bev", {})     # math family -> executor, or None: the torch modules run
        family = "f16" if self.math in F16_MATHS else "tf32x3"
        if family not in cache:
            if family == "f16":
                ok = hasattr(self.backbone, "forward_planes") and bev.rpn_is_fusable16(self.neck)
                stack = bev.FusedBevStack
            else:
                ok = hasattr(self.backbone, "forward_rows") and bev.rpn_is_fusable(self.neck)
                stack = bev.FusedBevStackTF32
            cache[family] = stack(self.neck, self.bbox_head) if ok else None
        return cache[family]


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
        if bev is not None:
            feats = self.reader(data["features"], data["num_voxels"])
            # the BEV map in the form the math's stack takes: f16 planes, or fp32 channels-last features
            f16 = self.math in F16_MATHS
            ovf = self.overflow_flag(feats.device) if f16 else None
            bev_input = self.backbone.forward_planes if f16 else self.backbone.forward_rows
            x = bev_input(feats, data["coors"], data["batch_size"], data["input_shape"], n_dev=data["n_dev"],
                          overflow=ovf)
            preds = bev.run(x, overflow=ovf)
        else:
            preds = self.bbox_head(self.extract_feat(data))
        if return_loss:
            return self.bbox_head.loss(example, preds)
        if kwargs.get("device_output", False):
            return self.bbox_head.predict_device(example, preds, self.test_cfg)
        return self.bbox_head.predict(example, preds, self.test_cfg)
