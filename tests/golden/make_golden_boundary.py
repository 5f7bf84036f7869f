"""Golden data for the boundary tests, produced by the REFERENCE itself.

Run with a Det3D reference checkout (V2AI/Det3D @ 230bb199) at REF (default ../reference beside the repository, or
the first argument):

    python tests/golden/make_golden_boundary.py [REF]

* reference_configs.json.gz -- the three stock configs as `Config.fromfile` parses the reference's own files: every key,
  tuples / ranges / loggers / the built box coder tagged so they come back as such (functions are recorded by name only; no test calls them).
* collate_kitti_reference.npz -- `collate_kitti` of the reference (det3d/torchie/parallel/collate.py:90-150), lifted out
  of its module, applied to the fixed batch of tests/test_pipeline_boundary.py::_sample.
* aot_voxel_reference.json -- digests of the reference's own voxelizer kernel (AOT-compiled into oracle/_ref) on the
  edge-case clouds of tests/boundary_golden.py::aot_voxel_cases.
* live_voxel_reference.npz -- `points_to_voxel` of the reference (det3d/ops/point_cloud/point_cloud_ops.py) on the three
  seeded clouds of tests/test_oracle_voxel.py::test_c_oracle_matches_live_reference_on_fresh_seeds.
"""
import ast
import collections
import gzip
import importlib.util
import json
import logging
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

STOCK = [
    "examples/second/configs/kitti_car_vfev3_spmiddlefhd_rpn1_mghead_syncbn.py",
    "examples/cbgs/configs/nusc_all_vfev3_spmiddleresnetfhd_rpn2_mghead_syncbn.py",
    "examples/point_pillars/configs/kitti_point_pillars_mghead_syncbn.py",
]


def encode(v):
    """Config value -> JSON value; tuples, ranges, loggers and functions are tagged (see boundary_golden.decode)."""
    if isinstance(v, dict):
        return {k: encode(x) for k, x in v.items()}
    if isinstance(v, tuple):
        return {"__tuple__": [encode(x) for x in v]}
    if isinstance(v, list):
        return [encode(x) for x in v]
    if isinstance(v, range):
        return {"__range__": [v.start, v.stop, v.step]}
    if isinstance(v, logging.Logger):
        return {"__logger__": v.name}
    if type(v).__name__ == "GroundBox3dCoderTorch":       # `build_box_coder(box_coder)` inside the config
        return {"__box_coder__": dict(type="ground_box3d_coder", linear_dim=v.linear_dim, encode_angle_vector=v.vec_encode,
                                      n_dim=v.n_dim, norm_velo=v.norm_velo)}
    if callable(v):
        return {"__function__": getattr(v, "__name__", repr(v))}
    if isinstance(v, (np.generic,)):
        return v.item()
    json.dumps(v)                   # anything else must already be plain JSON
    return v


def reference_collate(ref):
    src = open(os.path.join(ref, "det3d/torchie/parallel/collate.py")).read()
    fn = next(n for n in ast.parse(src).body if isinstance(n, ast.FunctionDef) and n.name == "collate_kitti")
    ns = dict(np=np, torch=torch, collections=collections, defaultdict=collections.defaultdict)
    exec(compile(ast.Module(body=[fn], type_ignores=[]), "collate.py", "exec"), ns)
    return ns["collate_kitti"]


def main(ref):
    from det3d.torchie import Config
    from boundary_golden import flatten, voxel_clouds
    from test_pipeline_boundary import COLLATE_BATCH, _sample

    cfgs = {}
    for rel in STOCK:
        cfg = Config.fromfile(os.path.join(ref, rel))
        cfgs[rel] = {k: encode(cfg[k]) for k in cfg}
    with gzip.open(os.path.join(HERE, "reference_configs.json.gz"), "wt") as fh:
        json.dump(cfgs, fh, sort_keys=True)

    want = reference_collate(ref)([_sample(i, n) for i, n in enumerate(COLLATE_BATCH)])
    arrays, kinds = flatten(want)
    np.savez_compressed(os.path.join(HERE, "collate_kitti_reference.npz"), __kinds__=np.array(json.dumps(kinds)), **arrays)

    spec = importlib.util.spec_from_file_location("ref_pc_ops", os.path.join(ref, "det3d/ops/point_cloud/point_cloud_ops.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    out = {}
    for seed, (pts, vs, pcr, max_pts, max_vox) in enumerate(voxel_clouds()):
        for name, a in zip(("voxels", "coors", "num_points"), mod.points_to_voxel(pts, vs, pcr, max_pts, True, max_vox)):
            out["%s_%d" % (name, seed)] = a
    np.savez_compressed(os.path.join(HERE, "live_voxel_reference.npz"), **out)

    # the reference's numba kernel compiled ahead of time (oracle/_ref, oracle/build.py) on the larger edge-case clouds;
    # stored as digests (the arrays would be ~0.8 MB): the comparison stays bit-exact
    from oracle import build as oracle_build
    from oracle import voxel_ref
    from boundary_golden import aot_voxel_cases, digest

    oracle_build.build()
    want = [[digest(a) for a in voxel_ref.points_to_voxel(pts, vs, pcr, max_pts, True, max_vox)]
            for pts, vs, pcr, max_pts, max_vox in aot_voxel_cases()]
    with open(os.path.join(HERE, "aot_voxel_reference.json"), "w") as fh:
        json.dump(want, fh, indent=1)
    for f in ("reference_configs.json.gz", "collate_kitti_reference.npz", "live_voxel_reference.npz", "aot_voxel_reference.json"):
        print(f, os.path.getsize(os.path.join(HERE, f)), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(os.path.dirname(ROOT), "reference"))
