"""d3b_predict_task (csrc/predict.cu + nms_batched in csrc/nms.cu) against a plain restatement of the reference's
get_task_detections (oracle/predict_cpu.py: predict_task_reference, mg_head.py:984-1085), across its parameter space.

Every draw is made decision-robust and the generator FAILS when one is not: passing scores are >= 1e-6 apart and from
the threshold, no pair entering NMS has an IoU within 1e-4 of the NMS threshold, no centre is within 1e-4 of a range
bound and no angle within 1e-5 of the direction offset (except values placed exactly there, which both sides compute
bit-exactly).  The device must then give exactly the oracle's detections: the same anchors in the same order, the same
labels, validity and count.  Scores must be bit-equal to torch.sigmoid run on the GPU (the reference's own op), boxes
bit-equal to the fp32 torch-op decode on the GPU and within a few ulps of a float64 decode.

Selection edges are checked against the reference's rule or the documented one: labels are the first class with the
maximal fp32 score, an anchor with a NaN logit is never emitted under a positive threshold, -0 and +0 are one logit,
ties in the logit go to the lower anchor index, and the set entering NMS is exactly {torch.sigmoid(x) >= threshold}."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

EPS32 = float(np.finfo(np.float32).eps)
PI4 = float(np.float32(np.pi / 4))
GAP_SCORE, GAP_IOU, GAP_RANGE, GAP_ANGLE = 1e-6, 1e-4, 1e-4, 1e-5


# ------------------------------------------------------------------------------------------------ generation (CPU)
def _logit(s):
    s = np.asarray(s, np.float64)
    return np.log(s / (1.0 - s)).astype(np.float32)


def _top_scores(rng, A, thr, n_pass):
    """Target top-class scores: n_pass anchors in [thr + 2e-4, 0.999], the rest in [2e-4, thr - 2e-4], every set
    rank-spaced (neighbours at least half a rank step apart) and shuffled over the anchors."""
    s = np.empty(A, np.float64)
    perm = rng.permutation(A)

    def spread(n, lo, hi):
        return lo + (hi - lo) * (rng.permutation(n) + rng.uniform(0.25, 0.75, n)) / max(n, 1)

    s[perm[:n_pass]] = spread(n_pass, (thr if thr > 0 else 0.0) + 2e-4, 0.999)
    s[perm[n_pass:]] = spread(A - n_pass, 2e-4, (thr if 0 < thr < 1 else 1.0) - 2e-4)
    return s


def _rot_iou_pairs(boxes):
    """IoU (rotate_nms_cc semantic, the C oracle) of every pair of [x, y, w, l, r] boxes whose circumscribed discs
    meet; every other pair has IoU 0."""
    from oracle.second_cpu import _nms_lib
    lib = _nms_lib()
    f = lib.oracle_rotate_iou_xywlr
    f.restype, f.argtypes = C.c_float, [C.c_void_p, C.c_void_p]
    b = np.ascontiguousarray(boxes, np.float32)
    r = 0.5 * np.hypot(b[:, 2], b[:, 3]) + 1e-3
    d = np.hypot(b[:, None, 0] - b[None, :, 0], b[:, None, 1] - b[None, :, 1])
    ii, jj = np.nonzero(np.triu(d <= r[:, None] + r[None, :], 1))
    return ii, np.array([f(b[i].ctypes.data, b[j].ctypes.data) for i, j in zip(ii, jj)], np.float64)


def _check_robust(name, R, enc, anchors, cfg, exact_r, exact_range):
    """Fail (never skip) when the draw leaves a decision within rounding of its boundary."""
    from oracle.aa_nms import iou_pixel_matrix
    from oracle.predict_cpu import second_box_decode
    thr, nd = cfg["thr"], cfg["nd"]
    nin = R["nms_in"]
    if nin.shape[0] == 0:
        return
    s = np.sort(R["all_scores"][R["all_scores"] >= thr] if thr > 0 else R["all_scores"])
    assert np.all(np.diff(s) >= GAP_SCORE), "%s: passing scores closer than %g" % (name, GAP_SCORE)
    if thr > 0:
        assert np.all(np.abs(R["all_scores"] - thr) >= GAP_SCORE), "%s: a score within %g of the threshold" % (name, GAP_SCORE)
    # NMS decides a pair when its higher-scored box is kept (nms_in is in descending score order)
    kept = np.isin(nin, R["anchor"])
    if cfg["iou"] <= 1.0:
        if cfg["rot"]:
            first, iou = _rot_iou_pairs(R["nms_boxes"])
            iou = iou[kept[first]]
        else:
            m = iou_pixel_matrix(R["nms_boxes"])
            iou = np.triu(m, 1)[kept][np.triu(np.ones_like(m, bool), 1)[kept]]
        assert not np.any(np.abs(iou - cfg["iou"]) < GAP_IOU), "%s: a pair's IoU is within %g of %g" % (
            name, GAP_IOU, cfg["iou"])
    # the direction flip and the range mask apply to the kept boxes
    sel = R["anchor"]
    b64 = second_box_decode(torch.from_numpy(enc[sel]).double(), torch.from_numpy(anchors[sel]).double(),
                            cfg["vec"], cfg["smooth"], cfg["norm_velo"]).numpy()
    if cfg["dir"]:
        d = np.abs(b64[:, nd - 1] - cfg["offset"])
        assert np.all((d >= GAP_ANGLE) | exact_r[sel]), "%s: an angle within %g of the offset" % (name, GAP_ANGLE)
    if cfg["range"] is not None:
        for c in range(3):
            for v in (cfg["range"][c], cfg["range"][3 + c]):
                d = np.abs(b64[:, c] - np.float32(v))
                assert np.all((d >= GAP_RANGE) | exact_range[sel, c]), "%s: a centre within %g of a bound" % (
                    name, GAP_RANGE)


def _gen_task(seed, B, hw, na, n_cls, nd, vec=False, smooth=False, norm_velo=False, dir=False, offset=0.0, rot=True,
              iou=0.5, thr=0.3, pre=1000, post=1000, has_range=False, label_offset=0, center_range=None):
    """Head, anchors and the oracle's detections of every sample, checked for decision robustness."""
    from oracle.predict_cpu import predict_task_reference
    rng = np.random.default_rng(seed)
    A = hw * na
    code = nd + (1 if vec else 0)
    cfg = dict(B=B, hw=hw, na=na, n_cls=n_cls, nd=nd, code=code, vec=vec, smooth=smooth, norm_velo=norm_velo, dir=dir,
               offset=offset, rot=rot, iou=iou, thr=thr, pre=pre, post=post, label_offset=label_offset)
    if thr <= 0:
        n_pass = [A] * B
    elif thr >= 0.999:
        n_pass = [0] * B
    else:
        n_pass = [int(rng.integers(min(A, max(1, pre // 3)), min(A, 2 * pre) + 1)) for _ in range(B)]
    n_in = max(1, min(pre, max(n_pass)))
    L = float(np.sqrt(n_in * 60.0)) + 10.0
    anchors = np.zeros((A, nd), np.float32)
    anchors[:, 0] = rng.uniform(0.0, L, A)
    anchors[:, 1] = rng.uniform(-L / 2, L / 2, A)
    anchors[:, 2] = rng.uniform(-2.0, 0.0, A)
    anchors[:, 3] = rng.uniform(1.5, 2.5, A)
    anchors[:, 4] = rng.uniform(3.5, 4.5, A)
    anchors[:, 5] = rng.uniform(1.3, 1.7, A)
    if nd == 9:
        anchors[:, 6:8] = rng.normal(size=(A, 2))
    near = rng.random(A) < 0.5
    anchors[:, nd - 1] = np.where(near, offset + rng.uniform(-0.6, 0.6, A), rng.uniform(-np.pi, np.pi, A))
    logits = np.empty((B, A, n_cls), np.float32)
    enc = np.empty((B, A, code), np.float32)
    dirs = np.empty((B, A, 2), np.float32)
    exact_r = np.zeros((B, A), bool)
    exact_range = np.zeros((B, A, 3), bool)
    rng_box = None
    if has_range:
        rng_box = [float(np.float32(v)) for v in (center_range or (0.1 * L, -0.4 * L, -1.6, 0.9 * L, 0.4 * L, -0.3))]
    for b in range(B):
        top = _logit(_top_scores(rng, A, thr, n_pass[b]))
        lab = rng.integers(0, n_cls, A)
        lg = (top[:, None] - rng.uniform(1.0, 4.0, (A, n_cls))).astype(np.float32)
        lg[np.arange(A), lab] = top
        logits[b] = lg
        e = np.empty((A, code), np.float32)
        e[:, :6] = rng.normal(0.0, 0.1, (A, 6))
        if nd == 9:
            e[:, 6:8] = rng.normal(0.0, 0.3, (A, 2))
        if vec:
            e[:, code - 2:] = rng.normal(0.0, 0.15, (A, 2))
        else:
            e[:, code - 1] = rng.normal(0.0, 0.3, A)
        enc[b] = e
        dirs[b] = rng.normal(size=(A, 2))
        tie = rng.random(A) < 0.05
        dirs[b, tie, 1] = dirs[b, tie, 0]                                   # exact ties: label 0, first maximum
        passing = np.nonzero(top >= _logit(thr) if thr > 0 else np.ones(A, bool))[0]
        if passing.shape[0] == 0:
            continue
        pick = rng.permutation(passing)
        if dir and not vec:                                                  # angles exactly on the offset
            for i in pick[:8]:
                anchors[i, nd - 1] = np.float32(offset)
                enc[b, i, code - 1] = 0.0
                exact_r[b, i] = True
        if has_range:                                                        # centres exactly on the inclusive bounds
            for t, i in enumerate(pick[8:20]):
                c, hi = t % 3, (t // 3) % 2
                anchors[i, c] = np.float32(rng_box[3 * hi + c])
                enc[b, i, c] = 0.0
                exact_range[b, i, c] = True
    cfg["range"] = rng_box
    want = []
    for b in range(B):
        R = predict_task_reference(torch.from_numpy(logits[b]), torch.from_numpy(enc[b]),
                                   torch.from_numpy(dirs[b]) if dir else None, torch.from_numpy(anchors), thr, pre, post,
                                   iou, rot, rng_box, offset, vec, smooth, norm_velo)
        top_s = torch.sigmoid(torch.from_numpy(logits[b])).max(-1)[0].numpy()
        R["all_scores"] = top_s
        R["nms_scores"] = top_s[R["nms_in"]]
        # an anchor whose angle was placed on the offset by another sample's draw is exact in this sample only if
        # its encoding is zero here as well
        _check_robust("sample %d" % b, R, enc[b], anchors, cfg,
                      exact_r[b] & (enc[b, :, code - 1] == 0.0) if (dir and not vec) else exact_r[b],
                      exact_range[b] & (enc[b, :, :3] == 0.0))
        want.append(R)
    return dict(cfg=cfg, logits=logits, enc=enc, dirs=dirs if dir else None, anchors=anchors, want=want)


# --------------------------------------------------------------------------------------------------- device side
def _lib():
    from det3d_b200 import _lib as L
    return L


def _strided(x, col0, pad):
    """[B, hw, w] values -> a NaN-filled [B, hw, col0 + w + pad] buffer holding them at column col0."""
    B, hw, w = x.shape
    buf = torch.full((B, hw, col0 + w + pad), float("nan"), device="cuda")
    buf[:, :, col0:col0 + w] = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    return buf


class _Dev:
    """Device buffers of one generated task, as column slices of wider fused rows (NaN in the other columns)."""

    def __init__(self, T, cls_col0=0, box_col0=0, dir_col0=0, pad=0):
        c = T["cfg"]
        B, hw, na = c["B"], c["hw"], c["na"]
        self.cls = _strided(T["logits"].reshape(B, hw, na * c["n_cls"]), cls_col0, pad)
        self.box = _strided(T["enc"].reshape(B, hw, na * c["code"]), box_col0, pad)
        self.dir = _strided(T["dirs"].reshape(B, hw, na * 2), dir_col0, pad) if T["dirs"] is not None else None
        self.anchors = torch.from_numpy(T["anchors"]).cuda()
        self.col0 = (cls_col0, box_col0, dir_col0)
        self.cfg = c

    def params(self):
        L, c = _lib(), self.cfg
        q = L.PredictParams()
        q.cls, q.cls_row_stride, q.cls_col0 = self.cls.data_ptr(), self.cls.shape[-1], self.col0[0]
        q.box, q.box_row_stride, q.box_col0 = self.box.data_ptr(), self.box.shape[-1], self.col0[1]
        if self.dir is not None:
            q.dir, q.dir_row_stride, q.dir_col0 = self.dir.data_ptr(), self.dir.shape[-1], self.col0[2]
        else:
            q.dir, q.dir_row_stride, q.dir_col0 = None, 0, 0
        q.anchors = self.anchors.data_ptr()
        q.batch, q.hw, q.na, q.n_cls, q.code, q.nd = c["B"], c["hw"], c["na"], c["n_cls"], c["code"], c["nd"]
        q.vec_encode, q.smooth_dim, q.norm_velo = int(c["vec"]), int(c["smooth"]), int(c["norm_velo"])
        q.use_rotate_nms, q.pre_max, q.post_max = int(c["rot"]), c["pre"], c["post"]
        q.nms_iou_threshold, q.score_threshold, q.direction_offset = c["iou"], c["thr"], c["offset"]
        q.has_range = 1 if c["range"] is not None else 0
        for k in range(6):
            q.post_center_range[k] = c["range"][k] if c["range"] is not None else 0.0
        q.label_offset = c["label_offset"]
        return q


def _workspace(q, fill=0):
    n = _lib().lib().d3b_predict_workspace_bytes(C.byref(q))
    return torch.full((n,), fill, dtype=torch.uint8, device="cuda")


def _call(q, packed, row_offset, counts, ws):
    L = _lib()
    st = L.lib().d3b_predict_task(C.byref(q), packed.data_ptr(), packed.shape[1], row_offset,
                                  counts.data_ptr() if counts is not None else None, ws.data_ptr(), ws.numel(),
                                  torch.cuda.current_stream().cuda_stream)
    L.check(st, "d3b_predict_task")


def _run(dev, rows=None, row_offset=0, ws=None, packed=None):
    c = dev.cfg
    q = dev.params()
    if packed is None:
        packed = torch.zeros((c["B"], rows or c["post"], c["nd"] + 3), device="cuda")
    counts = torch.full((c["B"],), -1, dtype=torch.int32, device="cuda")
    _call(q, packed, row_offset, counts, ws if ws is not None else _workspace(q))
    torch.cuda.synchronize()
    return packed, counts


def _bits(t):
    return t.contiguous().view(torch.int32).cpu().numpy()


def _decode_tol(enc, anc, cfg, flipped_angle):
    """A few fp32 ulps of the largest intermediate term of every decoded value (box_torch_ops.py:80-148)."""
    e, a = enc.astype(np.float64), anc.astype(np.float64)
    nd, q = cfg["nd"], (8 if cfg["nd"] == 9 else 6)
    diag = np.hypot(a[:, 3], a[:, 4])
    m = np.zeros((e.shape[0], nd))
    m[:, 0] = np.abs(e[:, 0]) * diag + np.abs(a[:, 0])
    m[:, 1] = np.abs(e[:, 1]) * diag + np.abs(a[:, 1])
    m[:, 2] = np.abs(e[:, 2]) * a[:, 5] + np.abs(a[:, 2])
    for k, (t, s) in enumerate(((3, 3), (4, 4), (5, 5))):
        m[:, k + 3] = ((np.abs(e[:, t]) + 1.0) if cfg["smooth"] else np.exp(e[:, t])) * a[:, s]
    if nd == 9:
        for k in (6, 7):
            m[:, k] = np.abs(e[:, k]) * (diag if cfg["norm_velo"] else 1.0) + np.abs(a[:, k])
    if cfg["vec"]:
        radius = np.hypot(e[:, q] + np.cos(a[:, nd - 1]), e[:, q + 1] + np.sin(a[:, nd - 1]))
        m[:, nd - 1] = (np.abs(e[:, q]) + np.abs(e[:, q + 1]) + 2.0) / radius + np.pi
    else:
        m[:, nd - 1] = np.abs(e[:, q]) + np.abs(a[:, nd - 1])
    m[:, nd - 1] += np.abs(flipped_angle) + np.pi
    return 4.0 * EPS32 * m


def _check_task(T, packed, counts, row_offset=0, counts_known=True):
    """Rows [row_offset, row_offset + post) of every sample against the oracle."""
    from oracle.predict_cpu import second_box_decode
    c = T["cfg"]
    nd, post = c["nd"], c["post"]
    logits = torch.from_numpy(T["logits"]).cuda()
    enc = torch.from_numpy(T["enc"]).cuda()
    anchors = torch.from_numpy(T["anchors"]).cuda()
    for b, R in enumerate(T["want"]):
        K = R["anchor"].shape[0]
        if counts_known:
            assert int(counts[b]) == K, "sample %d: %d kept, the oracle keeps %d" % (b, int(counts[b]), K)
        rows = packed[b, row_offset:row_offset + post]
        assert not np.any(_bits(rows[K:])), "sample %d: rows past the kept count are not zero" % b
        idx = torch.from_numpy(R["anchor"]).cuda()
        lab = torch.from_numpy(R["labels"]).cuda()
        got = rows[:K]
        assert np.array_equal(got[:, nd + 1].cpu().numpy(), R["labels"] + c["label_offset"]), "sample %d: labels" % b
        assert np.array_equal(got[:, nd + 2].cpu().numpy() > 0.5, R["valid"]), "sample %d: range mask" % b
        # scores: torch.sigmoid on the GPU, the reference's op, on the chosen class's logit
        want_s = torch.sigmoid(logits[b, idx, lab]) if K else got[:, nd]
        assert np.array_equal(_bits(got[:, nd]), _bits(want_s)), "sample %d: scores not bit-equal" % b
        # boxes: the fp32 torch-op decode and direction flip on the GPU, bit for bit (the same anchors, same order)
        want_b = second_box_decode(enc[b, idx], anchors[idx], c["vec"], c["smooth"], c["norm_velo"])
        if T["dirs"] is not None and K:
            dl = torch.max(torch.from_numpy(T["dirs"][b]).cuda()[idx], dim=-1)[1]
            opp = ((want_b[..., -1] - c["offset"]) > 0) ^ dl.bool()
            want_b[..., -1] += torch.where(opp, torch.tensor(np.pi).type_as(want_b), torch.tensor(0.0).type_as(want_b))
        assert np.array_equal(_bits(got[:, :nd]), _bits(want_b)), "sample %d: boxes not bit-equal to the torch decode" % b
        tol = _decode_tol(T["enc"][b][R["anchor"]], T["anchors"][R["anchor"]], c, R["boxes64"][:, nd - 1])
        err = np.abs(got[:, :nd].double().cpu().numpy() - R["boxes64"])
        assert np.all(err <= tol), "sample %d: decode error %g beyond the fp32 bound" % (b, float((err - tol).max()))


# ---------------------------------------------------------------------------------------------- parameter sweep
SWEEP = {
    # name: generator arguments (+ column layout)
    "second_point": dict(seed=1, B=1, hw=35200, na=2, n_cls=1, nd=7, dir=True, rot=True, iou=0.01, thr=0.3, pre=1000,
                         post=1000, has_range=True),
    "a_odd_vec_offset": dict(seed=2, B=3, hw=1037, na=1, n_cls=2, nd=7, vec=True, dir=True, offset=PI4, rot=True,
                             iou=0.5, thr=0.05, pre=1000, post=1, layout=(3, 2, 1, 5)),
    "small_nd9_smooth_norm": dict(seed=3, B=8, hw=200, na=2, n_cls=3, nd=9, vec=True, smooth=True, norm_velo=True,
                                  rot=False, iou=0.5, thr=0.3, pre=83, post=83, has_range=True),
    "pre_eq_a_1280_ten_cls": dict(seed=4, B=3, hw=1280, na=1, n_cls=10, nd=9, dir=True, offset=PI4, rot=True, iou=0.5,
                                  thr=0.0, pre=1280, post=1280, layout=(7, 1, 4, 3)),
    "pre_1279_pixel": dict(seed=101, B=3, hw=1279, na=1, n_cls=2, nd=7, smooth=True, dir=True, rot=False, iou=0.01,
                           thr=0.05, pre=1279, post=1279),
    "pre_2048_unstaged": dict(seed=104, B=1, hw=1024, na=2, n_cls=1, nd=9, vec=True, norm_velo=True, rot=True, iou=0.01,
                              thr=0.0, pre=2048, post=2048),
    "n_cls_255": dict(seed=7, B=3, hw=300, na=1, n_cls=255, nd=7, dir=True, rot=False, iou=2.0, thr=0.3, pre=1, post=1,
                      layout=(2, 0, 0, 9)),
    "nothing_passes": dict(seed=8, B=8, hw=2000, na=2, n_cls=2, nd=7, dir=True, rot=True, iou=0.5, thr=0.9999,
                           pre=1000, post=1000),
    "pre_1_no_filter": dict(seed=9, B=1, hw=400, na=1, n_cls=1, nd=7, rot=True, iou=2.0, thr=0.0, pre=1, post=1),
    "second_grid_pixel_2048": dict(seed=10, B=3, hw=35200, na=2, n_cls=2, nd=7, vec=True, dir=True, offset=PI4,
                                   rot=False, iou=0.5, thr=0.05, pre=2048, post=1, has_range=True, layout=(1, 1, 1, 1)),
    "pixel_1280_keep_all": dict(seed=11, B=1, hw=1500, na=2, n_cls=3, nd=7, dir=True, rot=False, iou=2.0, thr=0.3,
                                pre=1280, post=1280),
    "rot_2048_nd9": dict(seed=103, B=3, hw=3000, na=2, n_cls=1, nd=9, smooth=True, dir=True, rot=True, iou=0.5,
                         thr=0.05, pre=2048, post=2048, has_range=True),
    "rot_83_nd9_vec": dict(seed=13, B=8, hw=250, na=2, n_cls=2, nd=9, vec=True, dir=True, offset=PI4, rot=True,
                           iou=0.01, thr=0.3, pre=83, post=1),
}


def _make(name):
    args = dict(SWEEP[name])
    layout = args.pop("layout", (0, 0, 0, 0))
    return _gen_task(**args), layout


@pytest.mark.parametrize("name", sorted(SWEEP))
def test_predict_matches_reference(name):
    T, (c0, b0, d0, pad) = _make(name)
    dev = _Dev(T, c0, b0, d0, pad)
    packed, counts = _run(dev)
    _check_task(T, packed, counts)
    if T["cfg"]["thr"] >= 0.999:
        assert counts.tolist() == [0] * T["cfg"]["B"] and not torch.any(packed != 0)


# -------------------------------------------------------------------------------------------- adversarial selection
def _ident(logits, thr, pre, post=None, iou=2.0):
    """Anchor i sits at x = i with zero encodings, so a row's x IS its anchor index; at IoU threshold 2 NMS keeps every
    candidate and the rows list the selection in order.  logits [B, A, C] -> (anchor ids per sample, labels, scores)."""
    B, A, n_cls = logits.shape
    post = post or pre
    L = _lib()
    cls = logits.contiguous().cuda()
    box = torch.zeros((B, A, 7), device="cuda")
    anchors = torch.zeros((A, 7), device="cuda")
    anchors[:, 0] = torch.arange(A, device="cuda", dtype=torch.float32)
    anchors[:, 3:6] = 1.0
    q = L.PredictParams()
    q.cls, q.cls_row_stride, q.cls_col0 = cls.data_ptr(), n_cls, 0
    q.box, q.box_row_stride, q.box_col0 = box.data_ptr(), 7, 0
    q.dir = None
    q.anchors = anchors.data_ptr()
    q.batch, q.hw, q.na, q.n_cls, q.code, q.nd = B, A, 1, n_cls, 7, 7
    q.use_rotate_nms, q.pre_max, q.post_max = 1, pre, post
    q.nms_iou_threshold, q.score_threshold, q.has_range = iou, thr, 0
    packed = torch.zeros((B, post, 10), device="cuda")
    counts = torch.zeros(B, dtype=torch.int32, device="cuda")
    _call(q, packed, 0, counts, _workspace(q))
    torch.cuda.synchronize()
    out = []
    for b in range(B):
        k = int(counts[b])
        out.append((packed[b, :k, 0].long().cpu().numpy(), packed[b, :k, 8].long().cpu().numpy(), packed[b, :k, 7]))
    return out


@pytest.mark.parametrize("n_cls", [2, 3])
def test_label_is_first_class_with_the_maximal_score(n_cls):
    """Distinct logits that round to the same fp32 score, saturated (>= 17) and moderate (about 10): the label is the
    first class with the maximal score (mg_head.py:993, torch.max over the sigmoid scores), not the maximal logit."""
    g = torch.Generator().manual_seed(n_cls)
    A = 1200
    sat = 17.0 + 20.0 * torch.rand((A // 2, n_cls), generator=g)
    mod = 10.0 + 2e-3 * torch.rand((A // 2, n_cls), generator=g)
    logits = torch.cat([sat, mod]).unsqueeze(0)
    scores = torch.sigmoid(logits.cuda())
    want_lab = torch.max(scores, dim=-1)[1][0].cpu().numpy()
    want_s = torch.max(scores, dim=-1)[0][0]
    assert np.sum(want_lab != logits[0].argmax(-1).numpy()) >= A // 4       # the draw really has ties
    (ids, lab, sc), = _ident(logits, 0.5, A)
    assert sorted(ids.tolist()) == list(range(A))
    assert np.array_equal(lab, want_lab[ids])
    assert np.array_equal(_bits(sc), _bits(want_s[torch.from_numpy(ids).cuda()]))


@pytest.mark.parametrize("n_cls", [1, 2])
def test_nan_and_inf_logits(n_cls):
    """NaN in class 0 or in a later class: never emitted, and every passing anchor is still considered (pre_max is
    exactly the number that pass).  +inf scores 1 and passes; -inf never passes."""
    rng = np.random.default_rng(n_cls)
    A, P = 600, 150
    lg = rng.uniform(-6.0, -2.0, (A, n_cls)).astype(np.float32)
    perm = rng.permutation(A)
    good, nan0, nan1, pinf, ninf = perm[:P], perm[P:P + 60], perm[P + 60:P + 120], perm[P + 120:P + 130], perm[P + 130:P + 140]
    lg[good, 0] = rng.permutation(np.linspace(1.0, 3.0, P)).astype(np.float32)
    lg[nan0, 0] = np.nan
    if n_cls > 1:
        lg[nan0[:30], 1] = 8.0                  # NaN in class 0, a high later class
        lg[nan1, 0] = 8.0                       # a high class 0 and a NaN later: torch.max returns NaN
        lg[nan1, 1] = np.nan
    lg[pinf, n_cls - 1] = np.inf
    lg[ninf, :] = -np.inf
    want = set(good.tolist()) | set(pinf.tolist())
    (ids, lab, sc), = _ident(torch.from_numpy(lg).unsqueeze(0), 0.3, len(want))
    assert set(ids.tolist()) == want and ids.shape[0] == len(want)
    assert not torch.isnan(sc).any()
    s = sc.cpu().numpy()
    assert np.all(s[np.isin(ids, pinf)] == 1.0)


@pytest.mark.parametrize("A", [3000, 20000])
def test_signed_zero_logits_tie_by_index(A):
    """A plateau of alternating +0 / -0 logits larger than pre_max: one logit, so the lowest anchor indices win, in
    index order (A = 20000 exceeds the sort capacity: the radix select over composites)."""
    lg = torch.zeros((1, A, 1))
    lg[0, 1::2, 0] = -0.0
    assert torch.signbit(lg).sum() == A // 2
    (ids, _, sc), = _ident(lg, 0.3, 1000)
    assert ids.tolist() == list(range(1000))
    assert torch.all(sc == 0.5)


@pytest.mark.parametrize("thr", [0.05, 0.3, 0.7, 0.9])
def test_threshold_boundary_window(thr):
    """Every consecutive fp32 logit within +-256 ulps of logit(thr), shuffled over the anchors: the set entering NMS
    (IoU threshold 2 keeps all of it) is exactly {torch.sigmoid(x) >= thr} computed on the GPU."""
    x0 = np.float32(np.log(thr / (1.0 - thr)))
    bits = np.int64(x0.view(np.int32)) + np.arange(-256, 257)
    xs = bits.astype(np.int32).view(np.float32)
    assert np.all(np.sign(xs) == np.sign(x0)) or x0 == 0
    perm = np.random.default_rng(int(thr * 100)).permutation(xs.shape[0])
    lg = torch.from_numpy(xs[perm].copy()).reshape(1, -1, 1)
    passing = (torch.sigmoid(lg.cuda()) >= torch.tensor([thr], dtype=torch.float32, device="cuda"))[0, :, 0].cpu().numpy()
    assert 0 < passing.sum() < passing.shape[0]
    (ids, _, _), = _ident(lg, thr, xs.shape[0])
    assert set(ids.tolist()) == set(np.nonzero(passing)[0].tolist()) and ids.shape[0] == int(passing.sum())


@pytest.mark.parametrize("pre", [1000, 2048])
def test_radix_select_on_distinct_logits_in_one_bin(pre):
    """Sample 0: 20000 logits in [1, 1.25) (one 11-bit key bin, > 8192 candidates: the radix select) with some exact
    duplicates; in the same launch sample 1 takes the sorted path, nothing passes in sample 2, everything in sample 3.
    Every sample equals a stable host sort by (logit descending, index ascending), filtered by the threshold."""
    rng = np.random.default_rng(pre)
    A, thr = 20000, 0.3
    lo = np.float32(1.0).view(np.int32)
    x0 = (lo + rng.choice(1 << 21, A, replace=False)).astype(np.int32).view(np.float32)
    dup = rng.choice(A, 2000, replace=False)
    x0[dup[:1000]] = x0[dup[1000:]]
    lg = np.stack([x0, rng.normal(0.0, 3.0, A), rng.uniform(-6.0, -2.0, A), rng.uniform(2.0, 6.0, A)]).astype(np.float32)
    assert np.unique(x0).shape[0] > 8192
    got = _ident(torch.from_numpy(lg).unsqueeze(-1), thr, pre)
    passing = (torch.sigmoid(torch.from_numpy(lg).cuda()) >= torch.tensor([thr], device="cuda")).cpu().numpy()
    for b in range(4):
        order = np.lexsort((np.arange(A), -lg[b].astype(np.float64)))[:pre]
        want = order[passing[b, order]]
        assert np.array_equal(got[b][0], want), "sample %d" % b
    assert got[0][0].shape[0] == pre and got[2][0].shape[0] == 0 and got[3][0].shape[0] == pre


# ------------------------------------------------------------------------------------------------------- plumbing
def test_row_ranges_label_offset_and_two_tasks_in_one_buffer():
    """Two tasks write disjoint row ranges of one NaN-filled `packed`: rows outside [row_offset, row_offset + post)
    stay untouched, rows past keep_count are zero, label_offset is added; each range equals a standalone call."""
    T1 = _gen_task(21, B=3, hw=700, na=2, n_cls=2, nd=7, dir=True, rot=True, iou=0.5, thr=0.3, pre=200, post=60)
    T2 = _gen_task(22, B=3, hw=500, na=2, n_cls=3, nd=7, rot=False, iou=0.5, thr=0.3, pre=100, post=100, label_offset=7)
    d1, d2 = _Dev(T1), _Dev(T2)
    packed = torch.full((3, 190, 10), float("nan"), device="cuda")
    c1 = torch.full((3,), -1, dtype=torch.int32, device="cuda")
    c2 = torch.full((3,), -1, dtype=torch.int32, device="cuda")
    _call(d1.params(), packed, 10, c1, _workspace(d1.params()))
    _call(d2.params(), packed, 80, c2, _workspace(d2.params()))
    torch.cuda.synchronize()
    assert torch.isnan(packed[:, :10]).all() and torch.isnan(packed[:, 70:80]).all() and torch.isnan(packed[:, 180:]).all()
    _check_task(T1, packed, c1, row_offset=10)
    _check_task(T2, packed, c2, row_offset=80)
    assert int(c2.max()) < 100                                           # rows past keep_count were zeroed
    alone1, _ = _run(d1)
    alone2, _ = _run(d2)
    assert np.array_equal(_bits(packed[:, 10:70]), _bits(alone1)) and np.array_equal(_bits(packed[:, 80:180]), _bits(alone2))


def test_dirty_workspace_and_reuse():
    """A workspace full of 0xFF bytes gives what a zeroed one gives; a second call with other inputs on the same
    workspace equals a call on a fresh one."""
    Ta = _gen_task(31, B=3, hw=2000, na=2, n_cls=2, nd=7, dir=True, rot=True, iou=0.5, thr=0.3, pre=1000, post=100)
    Tb = _gen_task(32, B=3, hw=2000, na=2, n_cls=2, nd=7, dir=True, rot=True, iou=0.5, thr=0.3, pre=1000, post=100)
    da, db = _Dev(Ta), _Dev(Tb)
    dirty = _workspace(da.params(), 0xFF)
    pa_dirty, ca_dirty = _run(da, ws=dirty)
    pa_clean, ca_clean = _run(da, ws=_workspace(da.params()))
    assert np.array_equal(_bits(pa_dirty), _bits(pa_clean)) and torch.equal(ca_dirty, ca_clean)
    _check_task(Ta, pa_dirty, ca_dirty)
    pb_reused, cb_reused = _run(db, ws=dirty)
    pb_fresh, cb_fresh = _run(db, ws=_workspace(db.params()))
    assert np.array_equal(_bits(pb_reused), _bits(pb_fresh)) and torch.equal(cb_reused, cb_fresh)
    _check_task(Tb, pb_reused, cb_reused)


def test_graph_replay_matches_eager():
    """One d3b_predict_task captured in a CUDA graph, replayed over three fillings of the same buffers: each replay
    equals the eager call bit for bit."""
    fills = [_gen_task(42 + i, B=3, hw=1500, na=2, n_cls=2, nd=9, vec=True, dir=True, offset=PI4, rot=True, iou=0.5,
                       thr=0.3, pre=1000, post=200, has_range=True) for i in range(3)]
    devs = [_Dev(T, 2, 1, 3, 2) for T in fills]
    eager = [_run(d) for d in devs]
    static = _Dev(fills[0], 2, 1, 3, 2)
    q = static.params()
    ws = _workspace(q)
    packed = torch.zeros((3, 200, 12), device="cuda")
    counts = torch.zeros(3, dtype=torch.int32, device="cuda")
    _call(q, packed, 0, counts, ws)                     # warm-up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        _call(q, packed, 0, counts, ws)
    for i, d in enumerate(devs):
        static.cls.copy_(d.cls)
        static.box.copy_(d.box)
        static.dir.copy_(d.dir)
        static.anchors.copy_(d.anchors)
        packed.fill_(float("nan"))
        counts.fill_(-1)
        g.replay()
        torch.cuda.synchronize()
        assert np.array_equal(_bits(packed), _bits(eager[i][0])) and torch.equal(counts, eager[i][1]), "filling %d" % i
        _check_task(fills[i], packed, counts)


def test_predict_device_three_tasks_on_fused_rows():
    """MultiGroupHead.predict_device on a three-task head whose cls / box tensors are column slices of one fused
    NaN-padded row tensor: every task's rows equal the oracle, labels offset by the classes of the tasks before it."""
    from det3d_b200.core.bbox.box_coders import GroundBox3dCoderTorch
    from det3d_b200.models.bbox_heads.mg_head import MultiGroupHead
    B, H, W = 2, 20, 25
    n_cls = [1, 2, 3]
    thr, pre, post, iou = 0.3, 500, 80, 0.2
    center_range = (-5.0, -60.0, -1.8, 120.0, 60.0, -0.2)
    head = MultiGroupHead(in_channels=8, tasks=[dict(class_names=["c%d" % j for j in range(n)]) for n in n_cls],
                          box_coder=GroundBox3dCoderTorch(vec_encode=True, n_dim=9), loss_aux=None).cuda().eval()
    tasks, widths = [], []
    for t, n in enumerate(n_cls):
        tasks.append(_gen_task(51 + t, B=B, hw=H * W, na=2 * n, n_cls=n, nd=9, vec=True, rot=True, iou=iou, thr=thr,
                               pre=pre, post=post, has_range=True, label_offset=sum(n_cls[:t]), center_range=center_range))
        widths += [2 * n * n, 2 * n * 10]
    fused = torch.full((B, H, W, sum(widths) + 3), float("nan"), device="cuda")
    preds, anchors, col = [], [], 1
    for t, n in enumerate(n_cls):
        T = tasks[t]
        cls = fused[..., col:col + 2 * n * n]
        cls.copy_(torch.from_numpy(T["logits"]).reshape(B, H, W, -1))
        col += 2 * n * n
        box = fused[..., col:col + 2 * n * 10]
        box.copy_(torch.from_numpy(T["enc"]).reshape(B, H, W, -1))
        col += 2 * n * 10
        preds.append(dict(cls_preds=cls, box_preds=box))
        anchors.append(torch.from_numpy(T["anchors"]).cuda().unsqueeze(0).expand(B, -1, -1))
    test_cfg = dict(score_threshold=thr, post_center_limit_range=center_range,
                    nms=dict(use_multi_class_nms=False, use_rotate_nms=True, nms_pre_max_size=pre,
                             nms_post_max_size=post, nms_iou_threshold=iou))
    det = head.predict_device(dict(anchors=anchors), preds, test_cfg)
    torch.cuda.synchronize()
    packed = det["packed"]
    assert packed.shape == (B, 3 * post, 12)
    for t, T in enumerate(tasks):
        _check_task(T, packed, None, row_offset=t * post, counts_known=False)
    assert sum(int(R["valid"].sum()) for T in tasks for R in T["want"]) >= 50
