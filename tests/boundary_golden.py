"""Access to the reference-generated boundary fixtures (tests/golden/make_golden_boundary.py): the stock configs as the
reference's files parse, and the flattening used to store / compare nested collate outputs exactly."""
import gzip
import json
import logging
import os

import numpy as np
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def decode(v):
    if isinstance(v, list):
        return [decode(x) for x in v]
    if isinstance(v, dict):
        if "__tuple__" in v:
            return tuple(decode(x) for x in v["__tuple__"])
        if "__range__" in v:
            return range(*v["__range__"])
        if "__logger__" in v:
            return logging.getLogger(v["__logger__"])
        if "__box_coder__" in v:
            from det3d.builder import build_box_coder

            return build_box_coder(v["__box_coder__"])
        if "__function__" in v:
            return None                 # recorded by name only
        return {k: decode(x) for k, x in v.items()}
    return v


def reference_config(rel):
    """Config of the reference's own file `rel` (e.g. examples/second/configs/...py), as Config.fromfile parsed it."""
    from det3d.torchie import Config

    with gzip.open(os.path.join(GOLDEN, "reference_configs.json.gz"), "rt") as fh:
        return Config(decode(json.load(fh)[rel]), filename=None)


def flatten(obj, path="", arrays=None, kinds=None):
    """Nested dict / list / tuple of tensors, arrays and plain values -> ({path: ndarray}, {path: kind}); two objects are
    equal (type, dtype, shape, every bit) iff their flattenings are."""
    arrays = {} if arrays is None else arrays
    kinds = {} if kinds is None else kinds
    if isinstance(obj, dict):
        kinds[path] = ["dict", sorted(obj)]
        for k in obj:
            flatten(obj[k], "%s/%s" % (path, k), arrays, kinds)
    elif isinstance(obj, (list, tuple)):
        kinds[path] = [type(obj).__name__, len(obj)]
        for i, x in enumerate(obj):
            flatten(x, "%s/%d" % (path, i), arrays, kinds)
    elif torch.is_tensor(obj):
        kinds[path] = ["tensor", str(obj.dtype)]
        arrays[path] = obj.numpy()
    elif isinstance(obj, np.ndarray):
        kinds[path] = ["ndarray", str(obj.dtype)]
        arrays[path] = obj
    else:
        kinds[path] = ["value", type(obj).__name__, json.loads(json.dumps(obj))]
    return arrays, kinds


def load_flat(name):
    g = np.load(os.path.join(GOLDEN, name))
    return {k: g[k] for k in g.files if k != "__kinds__"}, json.loads(str(g["__kinds__"]))


def aot_voxel_cases():
    """Seeded clouds ~1 m beyond the range, 30 % snapped to exact voxel-size multiples (fp32 division edge cases): KITTI
    SECOND, PointPillars (hits the max_voxels break), nuScenes ndim 5, an empty ndim-3 cloud.
    -> [(pts, voxel_size, range, max_points, max_voxels)]."""
    rng = np.random.default_rng(123)
    cases = [([0.05, 0.05, 0.1], [0, -40.0, -3.0, 70.4, 40.0, 1.0], 5, 20000, 4, 30000),
             ([0.16, 0.16, 4.0], [0, -39.68, -3, 69.12, 39.68, 1], 100, 1200, 4, 9000),
             ([0.1, 0.1, 0.2], [-51.2, -51.2, -5.0, 51.2, 51.2, 3.0], 10, 60000, 5, 20000),
             ([0.05, 0.05, 0.1], [0, -40.0, -3.0, 70.4, 40.0, 1.0], 5, 20000, 3, 0)]
    out = []
    for vs, pcr, max_pts, max_vox, ndim, n in cases:
        lo, hi = np.asarray(pcr[:3], np.float32), np.asarray(pcr[3:], np.float32)
        span = (hi - lo + 2.0)[[0, 1, 2] + [0] * (ndim - 3)]
        base = (lo - 1.0)[[0, 1, 2] + [0] * (ndim - 3)]
        pts = (base + rng.random((n, ndim)).astype(np.float32) * span).astype(np.float32)
        if n:
            snap = rng.random(n) < 0.3
            cell = np.floor((pts[snap, :3] - lo) / np.asarray(vs, np.float32))
            pts[snap, :3] = lo + cell * np.asarray(vs, np.float32)
        out.append((pts, vs, pcr, max_pts, max_vox))
    return out


def digest(a):
    """[shape, dtype, sha256 of the bytes]: equal iff the arrays are bit-identical."""
    import hashlib

    a = np.ascontiguousarray(a)
    return [list(a.shape), str(a.dtype), hashlib.sha256(a.tobytes()).hexdigest()]


def voxel_clouds():
    """The three seeded KITTI-range clouds (and voxelizer settings) of the live-reference voxel comparison."""
    rng = np.random.default_rng(123)
    vs, pcr = np.float32([0.05, 0.05, 0.1]), np.float32([0, -40, -3, 70.4, 40, 1])
    out = []
    for seed in range(3):
        n = int(rng.integers(100, 5000))
        pts = np.stack([rng.uniform(-1, 71, n), rng.uniform(-41, 41, n), rng.uniform(-3.2, 1.2, n), rng.uniform(0, 1, n)],
                       1).astype(np.float32)
        out.append((pts, vs, pcr, 5, 600 + 700 * seed))
    return out
