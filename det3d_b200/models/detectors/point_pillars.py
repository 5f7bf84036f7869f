"""PointPillars detector (det3d/models/detectors/point_pillars.py:5-54): PillarFeatureNet reader ->
PointPillarsScatter -> RPN -> MultiGroupHead."""
from ..registry import DETECTORS
from .voxelnet import F16_MATHS, SingleStageDetector, _FusedBevMixin


@DETECTORS.register_module
class PointPillars(_FusedBevMixin, SingleStageDetector):
    def _read(self, data):
        """Pillar features [rows, units]: through the voxelizer's point-index lists when the caller passes them (the
        [M, 100, ndim] voxel tensor is then never built -- SURVEY 8f.3), else from the materialised voxel tensor."""
        n_dev = data.get("n_dev")
        lists = data.get("point_lists")
        if lists is not None and n_dev is not None and hasattr(self.reader, "forward_lists") and not self.training:
            return self.reader.forward_lists(lists, data["num_voxels"], data["coors"], data["coors"].shape[0], n_dev)
        kw = {} if n_dev is None else {"n_dev": n_dev}
        return self.reader(data["features"], data["num_voxels"], data["coors"], **kw)

    def extract_feat(self, data):
        n_dev = data.get("n_dev")
        kw = {} if n_dev is None else {"n_dev": n_dev}
        feats = self._read(data)
        x = self.backbone(feats, data["coors"], data["batch_size"], data["input_shape"], **kw)
        return self.neck(x) if self.with_neck else x

    def forward(self, example, return_loss=True, **kwargs):
        num_voxels = example["num_voxels"]
        data = dict(features=example["voxels"], num_voxels=example["num_points"], coors=example["coordinates"],
                    batch_size=len(num_voxels), input_shape=example["shape"][0], n_dev=example.get("n_voxels_dev"),
                    point_lists=example.get("point_lists"))
        bev = self.fused_bev() if not return_loss else None
        if bev is not None and self.math in F16_MATHS:
            kw = {} if data["n_dev"] is None else {"n_dev": data["n_dev"]}
            feats = self._read(data)
            ovf = self.overflow_flag(feats.device)
            planes = self.backbone.forward_planes(feats, data["coors"], data["batch_size"], data["input_shape"],
                                                  overflow=ovf, n_planes=self.n_planes(), **kw)
            preds = bev.run(planes, overflow=ovf)
        else:
            preds = self.bbox_head(self.extract_feat(data))
        if return_loss:
            return self.bbox_head.loss(example, preds)
        if kwargs.get("device_output", False):
            return self.bbox_head.predict_device(example, preds, self.test_cfg)
        return self.bbox_head.predict(example, preds, self.test_cfg)
