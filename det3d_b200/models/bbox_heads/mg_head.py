"""MultiGroupHead: per-task 1x1 conv heads + device-resident `predict`.

Constructor, parameter names (`tasks.<i>.conv_box|conv_cls|conv_dir`), `forward` output
dicts and `predict(example, preds_dicts, test_cfg)` results follow
det3d/models/bbox_heads/mg_head.py:198-230, 386-533, 697-1085.  What changes is *where*
post-processing runs: the reference loops over samples in Python and ships the top-1000
boxes to a CPU NMS (box_torch_ops.py:537-541); here anchor decode, sigmoid, score
filter, top-k, rotated NMS (csrc/nms.cu), direction fix and range mask all stay on the
GPU with fixed-shape buffers, and `predict` only synchronises once, at the end, to
slice the variable-length results the API promises.  Loss code is training-only and
out of scope.
"""
import logging

import numpy as np
import torch
from torch import nn

from det3d_b200 import _lib
from det3d_b200.core.bbox import box_torch_ops
from det3d_b200.ops.nms import nms_ops

from ..builder import build_loss
from ..registry import HEADS


_TASK_STREAMS = {}     # device -> side streams the per-task predict chains are forked over


@HEADS.register_module
class Head(nn.Module):
    def __init__(self, num_input, num_pred, num_cls, use_dir=False, num_dir=0, header=True, name="",
                 focal_loss_init=False, **kwargs):
        super().__init__(**kwargs)
        self.use_dir = use_dir
        self.conv_box = nn.Conv2d(num_input, num_pred, 1)
        self.conv_cls = nn.Conv2d(num_input, num_cls, 1)
        if self.use_dir:
            self.conv_dir = nn.Conv2d(num_input, num_dir, 1)

    def forward(self, x):
        out = {
            "box_preds": self.conv_box(x).permute(0, 2, 3, 1).contiguous(),
            "cls_preds": self.conv_cls(x).permute(0, 2, 3, 1).contiguous(),
        }
        if self.use_dir:
            out["dir_cls_preds"] = self.conv_dir(x).permute(0, 2, 3, 1).contiguous()
        return out


class _PackedDetections(dict):
    """dict(packed, boxes, scores, labels, valid) over the packed device tensor; `labels` (int64) and `valid` (bool) are
    materialised on first access only -- the serving path ships `packed` as is and would pay two extra launches per step."""

    def __init__(self, packed, nd):
        super().__init__(packed=packed, boxes=packed[..., :nd], scores=packed[..., nd])
        self._nd = nd

    def __missing__(self, key):
        packed, nd = dict.__getitem__(self, "packed"), self._nd
        if key == "labels":
            value = packed[..., nd + 1].long()
        elif key == "valid":
            value = packed[..., nd + 2] > 0.5
        else:
            raise KeyError(key)
        self[key] = value
        return value

    def __contains__(self, key):
        return key in ("labels", "valid") or dict.__contains__(self, key)


@HEADS.register_module
class MultiGroupHead(nn.Module):
    def __init__(self, mode="3d", in_channels=[128], norm_cfg=None, tasks=[], weights=[], num_classes=[1],
                 box_coder=None, with_cls=True, with_reg=True, reg_class_agnostic=False,
                 encode_background_as_zeros=True, loss_norm=None, loss_cls=None, use_sigmoid_score=True,
                 loss_bbox=None, encode_rad_error_by_sin=True, loss_aux=None, direction_offset=0.0,
                 name="rpn", logger=None):
        super().__init__()
        assert with_cls or with_reg
        num_classes = [len(t["class_names"]) for t in tasks]
        self.class_names = [t["class_names"] for t in tasks]
        self.num_anchor_per_locs = [2 * n for n in num_classes]
        self.box_coder = box_coder
        self.with_cls, self.with_reg = with_cls, with_reg
        self.in_channels = in_channels
        self.num_classes = num_classes
        self.reg_class_agnostic = reg_class_agnostic
        self.encode_rad_error_by_sin = encode_rad_error_by_sin
        self.encode_background_as_zeros = encode_background_as_zeros
        self.use_sigmoid_score = use_sigmoid_score
        self.box_n_dim = box_coder.code_size
        self.anchor_dim = box_coder.n_dim
        if loss_cls is not None:
            self.loss_cls = build_loss(loss_cls)
        if loss_bbox is not None:
            self.loss_reg = build_loss(loss_bbox)
        if loss_aux is not None:
            self.loss_aux = build_loss(loss_aux)
        self.loss_norm = loss_norm
        self.logger = logger or logging.getLogger("MultiGroupHead")
        self.use_direction_classifier = loss_aux is not None
        self.direction_offset = direction_offset if loss_aux else 0.0
        self.bev_only = mode == "bev"

        self.tasks = nn.ModuleList()
        for n_cls, n_anchor in zip(num_classes, self.num_anchor_per_locs):
            num_cls = n_anchor * n_cls if encode_background_as_zeros else n_anchor * (n_cls + 1)
            code = box_coder.code_size - 2 if self.bev_only else box_coder.code_size
            self.tasks.append(Head(in_channels, n_anchor * code, num_cls, use_dir=self.use_direction_classifier,
                                   num_dir=n_anchor * 2 if self.use_direction_classifier else None, header=False))
        self.logger.info("Finish MultiGroupHead Initialization")

    def init_weights(self, pretrained=None):
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
                if m.bias is not None:
                    nn.init.constant_(m.bias, 0)

    def forward(self, x):
        return [task(x) for task in self.tasks]

    def loss(self, example, preds_dicts, **kwargs):
        raise NotImplementedError("training is out of scope for det3d_b200 (inference hot path only)")

    # ------------------------------------------------------------------ predict
    def _task_device_detections(self, task_id, test_cfg, cls_preds, box_preds, anchors, dir_preds):
        """One task, whole batch, fixed shapes, no host sync.

        cls_preds [B,A,C] logits, box_preds [B,A,code] encodings, anchors [B,A,nd], dir_preds [B,A,2] | None.
        -> boxes [B,P,nd], scores [B,P], labels [B,P] int64, valid [B,P] bool  (P = nms_post_max_size)

        Same selection as mg_head.py:995-1025 (score filter, then top-`nms_pre_max_size`), done as
        top-k first / filter second (sigmoid is monotonic, the passing set is a prefix of the top-k),
        so only the `pre` selected anchors are decoded instead of all 70,400."""
        nms_cfg = test_cfg["nms"] if isinstance(test_cfg, dict) else test_cfg.nms
        if nms_cfg["use_multi_class_nms"]:
            raise NotImplementedError("use_multi_class_nms=True is not used by the Det3D configs in scope")
        if not (self.encode_background_as_zeros and self.use_sigmoid_score):
            raise NotImplementedError("only sigmoid scores with background-as-zeros are on the hot path")
        B, A, C = cls_preds.shape
        dev = cls_preds.device
        thr = float(test_cfg["score_threshold"])
        pre = min(int(nms_cfg["nms_pre_max_size"]), A)
        post = min(int(nms_cfg["nms_post_max_size"]), pre)
        logits = cls_preds.float()
        if C == 1:
            top_logit, top_labels = logits.squeeze(-1), None
        else:
            # mg_head.py:993: the label is the first class with the maximal fp32 SCORE (distinct logits can share one)
            top_labels = torch.max(torch.sigmoid(logits), dim=-1)[1]
            top_logit = torch.gather(logits, -1, top_labels.unsqueeze(-1)).squeeze(-1)
        sel_logit, sel_idx = torch.topk(top_logit, k=pre, dim=1)                 # descending
        sel_scores = torch.sigmoid(sel_logit)
        if thr > 0.0:
            n_valid = (sel_scores >= thr).sum(dim=1).to(torch.int32)
        else:
            n_valid = torch.full((B,), pre, dtype=torch.int32, device=dev)
        nd = anchors.shape[-1]
        code = box_preds.shape[-1]
        enc = torch.gather(box_preds.float(), 1, sel_idx.unsqueeze(-1).expand(B, pre, code))
        anc = torch.gather(anchors.float(), 1, sel_idx.unsqueeze(-1).expand(B, pre, nd))
        cand = self.box_coder.decode_torch(enc[:, :, : self.box_coder.code_size], anc)   # [B,pre,nd]
        if self.use_direction_classifier and dir_preds is not None:
            dsel = torch.gather(dir_preds, 1, sel_idx.unsqueeze(-1).expand(B, pre, 2))
            dir_labels = torch.max(dsel, dim=-1)[1]
        lab = torch.zeros((B, pre), dtype=torch.long, device=dev) if top_labels is None else torch.gather(top_labels, 1, sel_idx)
        use_rot = bool(nms_cfg["use_rotate_nms"])
        slot = torch.arange(post, device=dev)
        keep_all, ok_all = [], []
        for b in range(B):
            if use_rot:
                cb = cand[b]   # (no list indexing: it would stage an index tensor through the host)
                nms_boxes = torch.stack([cb[:, 0], cb[:, 1], cb[:, 3], cb[:, 4], cb[:, nd - 1]], dim=1)
                keep_idx, keep_count = nms_ops.nms_sorted(nms_boxes, _lib.BOX_XYWLR,
                                                          float(nms_cfg["nms_iou_threshold"]), post,
                                                          n_dev=n_valid[b:b + 1])
            else:
                corners = box_torch_ops.center_to_corner_box2d(cand[b][:, :2], cand[b][:, 3:5], cand[b][:, nd - 1])
                bb = torch.cat([box_torch_ops.corner_to_standup_nd(corners),
                                torch.zeros((pre, 1), device=dev)], dim=1).contiguous()
                keep_idx, keep_count = nms_ops.nms_sorted(bb, _lib.BOX_XYXYR, float(nms_cfg["nms_iou_threshold"]),
                                                          post, n_dev=n_valid[b:b + 1], axis_aligned=True,
                                                          aa_mode=_lib.AA_PIXEL)
            ok = slot < keep_count.to(torch.long)
            keep_all.append(torch.where(ok, keep_idx[:post], torch.zeros_like(keep_idx[:post])))
            ok_all.append(ok)
        kidx = torch.stack(keep_all)                                              # [B,post]
        valid = torch.stack(ok_all)
        boxes = torch.gather(cand, 1, kidx.unsqueeze(-1).expand(B, post, nd))
        scores = torch.gather(sel_scores, 1, kidx)
        labels = torch.gather(lab, 1, kidx)
        if self.use_direction_classifier and dir_preds is not None:
            dl = torch.gather(dir_labels, 1, kidx)
            opp = ((boxes[..., -1] - self.direction_offset) > 0) ^ dl.bool()
            boxes = torch.cat([boxes[..., :-1], (boxes[..., -1] + opp.to(boxes.dtype) * np.pi).unsqueeze(-1)], -1)
        rng = test_cfg["post_center_limit_range"]
        if rng is not None and len(rng) > 0:
            key = (tuple(float(v) for v in rng), dev)
            cache = self.__dict__.setdefault("_range_cache", {})
            r = cache.get(key)
            if r is None:   # built once (a host->device copy is not CUDA-graph capturable)
                r = cache[key] = torch.tensor(list(rng), dtype=torch.float32, device=dev)
            valid = valid & (boxes[..., :3] >= r[:3]).all(-1) & (boxes[..., :3] <= r[3:]).all(-1)
        return boxes, scores, labels, valid

    def _check_supported(self, example, **kwargs):
        """Inputs the reference's predict treats specially and this path does not implement: fail, never differ."""
        if isinstance(example, dict) and example.get("anchors_mask") is not None:
            raise NotImplementedError("example['anchors_mask'] (pos_area_threshold >= 0, mg_head.py:760-767,983-993) is "
                                      "not implemented on the device predict path")
        if kwargs.get("mode") is not None:
            raise NotImplementedError("predict(mode=...) (bev_only path) is not implemented")
        seen = self.__dict__.setdefault("_anchor_batch_checked", set())
        for a in example["anchors"]:
            if a.dim() >= 3 and a.shape[0] > 1 and a.stride(0) != 0:
                key = (a.data_ptr(), a._version, tuple(a.shape))
                if key not in seen:      # one-time check per anchor tensor (synchronises once)
                    if not bool((a == a[:1]).all()):
                        raise NotImplementedError("per-sample anchors differ: the device predict path assumes one "
                                                  "anchor set per task shared by the batch")
                    seen.add(key)

    @staticmethod
    def _rows(t, batch):
        """[B,H,W,n] head tensor (contiguous or a column slice of fused rows) -> (ptr, row stride in floats, hw)."""
        assert t.dtype == torch.float32 and t.dim() == 4 and t.shape[0] == batch and t.stride(-1) == 1
        h, w = t.shape[1], t.shape[2]
        rs = t.stride(2)
        assert t.stride(1) == w * rs and (batch == 1 or t.stride(0) == h * w * rs), "head rows must be uniformly strided"
        return t.data_ptr(), rs, h * w

    def predict_device(self, example, preds_dicts, test_cfg, use_torch_ops=False):
        """Fixed-shape, sync-free detections for the whole batch.

        -> dict(packed [B,D,nd+3], boxes [B,D,nd], scores [B,D], labels [B,D] int64, valid [B,D] bool) with
        D = sum over tasks of nms_post_max_size; labels already offset per task.  One d3b_predict_task
        call (five kernels + NMS) per task; `use_torch_ops=True` runs the same algorithm with torch
        ops (kept as an in-repo cross-check of the fused kernels)."""
        self._check_supported(example)
        if use_torch_ops:
            return self._predict_device_torch(example, preds_dicts, test_cfg)
        import ctypes as C
        nms_cfg = test_cfg["nms"] if isinstance(test_cfg, dict) else test_cfg.nms
        if nms_cfg["use_multi_class_nms"]:
            raise NotImplementedError("use_multi_class_nms=True is not used by the Det3D configs in scope")
        if not (self.encode_background_as_zeros and self.use_sigmoid_score):
            raise NotImplementedError("only sigmoid scores with background-as-zeros are on the hot path")
        first = preds_dicts[0]["cls_preds"]
        dev, B = first.device, first.shape[0]
        nd = self.anchor_dim
        posts, D = [], 0
        for task_id in range(len(preds_dicts)):
            A = example["anchors"][task_id].reshape(B, -1, nd).shape[1]
            pre = min(int(nms_cfg["nms_pre_max_size"]), A)
            posts.append((pre, min(int(nms_cfg["nms_post_max_size"]), pre)))
            D += posts[-1][1]
        cache = self.__dict__.setdefault("_predict_bufs", {})
        key = (B, D, nd, dev)
        if key not in cache:
            cache[key] = dict(packed=torch.zeros((B, D, nd + 3), dtype=torch.float32, device=dev), ws={})
        bufs = cache[key]
        packed = bufs["packed"]
        rng = test_cfg["post_center_limit_range"]
        row_offset, flag = 0, 0
        calls = []
        for task_id, preds in enumerate(preds_dicts):
            pre, post = posts[task_id]
            q = _lib.PredictParams()
            q.cls, q.cls_row_stride, hw = self._rows(preds["cls_preds"], B)
            q.box, q.box_row_stride, _ = self._rows(preds["box_preds"], B)
            q.cls_col0 = q.box_col0 = q.dir_col0 = 0
            if self.use_direction_classifier:
                q.dir, q.dir_row_stride, _ = self._rows(preds["dir_cls_preds"], B)
            else:
                q.dir, q.dir_row_stride = None, 0
            anchors = example["anchors"][task_id].reshape(B, -1, nd)[0].contiguous()   # identical for every sample
            q.anchors = anchors.data_ptr()
            n_cls = self.num_classes[task_id]
            q.batch, q.hw, q.na, q.n_cls = B, hw, anchors.shape[0] // hw, n_cls
            q.code = self.box_n_dim - 2 if self.bev_only else self.box_n_dim
            q.nd = nd
            q.vec_encode = 1 if self.box_coder.vec_encode else 0
            # the reference's decode_torch never reaches smooth_dim / norm_velo (see box_coders.decode_torch)
            q.smooth_dim = 0
            q.norm_velo = 0
            q.use_rotate_nms = 1 if nms_cfg["use_rotate_nms"] else 0
            q.pre_max, q.post_max = pre, post
            q.nms_iou_threshold = float(nms_cfg["nms_iou_threshold"])
            q.score_threshold = float(test_cfg["score_threshold"])
            q.direction_offset = float(self.direction_offset)
            q.has_range = 1 if (rng is not None and len(rng) > 0) else 0
            for c in range(6):
                q.post_center_range[c] = float(rng[c]) if q.has_range else 0.0
            q.label_offset = flag
            need = _lib.lib().d3b_predict_workspace_bytes(C.byref(q))
            ws = bufs["ws"].get(task_id)
            if ws is None or ws.numel() < need:
                ws = bufs["ws"][task_id] = torch.empty(need, dtype=torch.uint8, device=dev)
            calls.append((q, ws, row_offset, dict(anchors=int(anchors.shape[0]), batch=B, pre=pre, post=post), anchors))
            row_offset += post
            flag += n_cls
        # The tasks are independent (own head columns, own workspace, own rows of `packed`) and each is a chain of small
        # launches: fork them over side streams so the chains overlap (CBGS: six tasks), join before anyone reads `packed`.
        # Everything the calls read was enqueued before the fork; inside a CUDA-graph capture this becomes a fork/join.
        main = torch.cuda.current_stream(dev)
        pool = _TASK_STREAMS.setdefault(dev, [])      # (module-level: the head must stay deep-copyable)
        while len(pool) < len(calls) - 1:
            pool.append(torch.cuda.Stream(device=dev))
        for side in pool[:len(calls) - 1]:
            side.wait_stream(main)
        for i, (q, ws, row0, info, _anchors) in enumerate(calls):
            stream = main if i == 0 else pool[i - 1]
            with torch.cuda.stream(stream), _lib.on_device_of(packed, first), _lib.timed("predict", **info):
                st = _lib.lib().d3b_predict_task(C.byref(q), packed.data_ptr(), D, row0, None, ws.data_ptr(), ws.numel(),
                                                _lib.current_stream())
            _lib.check(st, "d3b_predict_task")
        for side in pool[:len(calls) - 1]:
            main.wait_stream(side)
        return _PackedDetections(packed, nd)

    def _predict_device_torch(self, example, preds_dicts, test_cfg):
        outs = []
        flag = 0
        for task_id, preds in enumerate(preds_dicts):
            anchors = example["anchors"][task_id]
            B = anchors.shape[0]
            anchors = anchors.view(B, -1, self.anchor_dim)
            code = self.box_n_dim - 2 if self.bev_only else self.box_n_dim
            box_preds = preds["box_preds"].reshape(B, -1, code)
            n_cls = self.num_classes[task_id] if self.encode_background_as_zeros else self.num_classes[task_id] + 1
            cls_preds = preds["cls_preds"].reshape(B, -1, n_cls)
            dirs = preds["dir_cls_preds"].reshape(B, -1, 2) if self.use_direction_classifier else None
            bx, sc, lb, ok = self._task_device_detections(task_id, test_cfg, cls_preds, box_preds, anchors, dirs)
            outs.append((bx, sc, lb + flag, ok))
            flag += self.num_classes[task_id]
        return dict(boxes=torch.cat([o[0] for o in outs], 1), scores=torch.cat([o[1] for o in outs], 1),
                    labels=torch.cat([o[2] for o in outs], 1), valid=torch.cat([o[3] for o in outs], 1))

    def predict(self, example, preds_dicts, test_cfg, **kwargs):
        """list (per sample) of dict(box3d_lidar [K,nd], scores [K], label_preds [K], metadata)."""
        self._check_supported(example, **kwargs)
        det = self.predict_device(example, preds_dicts, test_cfg)
        B = det["boxes"].shape[0]
        meta = example.get("metadata") if isinstance(example, dict) else None
        if not meta:
            meta = [None] * B
        results = []
        for b in range(B):
            m = det["valid"][b]
            results.append({"box3d_lidar": det["boxes"][b][m], "scores": det["scores"][b][m],
                            "label_preds": det["labels"][b][m], "metadata": meta[b]})
        return results
