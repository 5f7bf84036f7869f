"""Golden data of the SECOND KITTI three-class and CBGS Lyft stock configs, produced by the REFERENCE itself.

Run with a Det3D reference checkout (V2AI/Det3D @ 230bb199) at REF (default ../reference beside the repository, or
the first argument):

    python tests/golden/make_golden_configs_more.py [REF]

* reference_configs_more.json.gz -- examples/second/configs/kitti_all_vfev3_spmiddlefhd_rpn1_mghead_syncbn.py and
  examples/cbgs/configs/lyft_all_vfev3_spmiddleresnetfhd_rpn2_mghead_syncbn.py as `Config.fromfile` parses them, encoded
  by make_golden_boundary.encode (the encoding of reference_configs.json.gz).  A file of its own, so that the existing
  fixtures stay byte-identical; the gzip header carries no timestamp.
* anchors_lyft.npz -- det3d/core/bbox/box_np_ops.py create_anchors_3d_range (function source exec'd in isolation, with
  the `list(...)` shim of make_golden.py for numpy >= 2) for each of the Lyft config's seven anchor generators on the
  [1, 252, 252] feature map: per class 512 seeded sample rows, the float64 sum and sum of squares, and the shape.
"""
import gzip
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)

from make_golden_boundary import encode  # noqa: E402  (also puts the repository root on sys.path)

STOCK = [
    "examples/second/configs/kitti_all_vfev3_spmiddlefhd_rpn1_mghead_syncbn.py",
    "examples/cbgs/configs/lyft_all_vfev3_spmiddleresnetfhd_rpn2_mghead_syncbn.py",
]
OUT = "reference_configs_more.json.gz"
LYFT_FEATURE_MAP = [1, 252, 252]


def reference_create_anchors(ref):
    src = open(os.path.join(ref, "det3d/core/bbox/box_np_ops.py")).read()
    fn = src[src.index("def create_anchors_3d_range"):src.index("def create_anchors_bev_range")]
    fn = fn.replace('indexing="ij")', 'indexing="ij")\n    rets = list(rets)')
    ns = {"np": np}
    exec(fn, ns)
    return ns["create_anchors_3d_range"]


def main(ref):
    from det3d.torchie import Config

    data = {}
    for rel in STOCK:
        cfg = Config.fromfile(os.path.join(ref, rel))
        data[rel] = {k: encode(cfg[k]) for k in cfg}
    with open(os.path.join(HERE, OUT), "wb") as raw, gzip.GzipFile(filename="", mode="wb", fileobj=raw, mtime=0) as gz:
        gz.write(json.dumps(data, sort_keys=True).encode())
    print(OUT, os.path.getsize(os.path.join(HERE, OUT)), "bytes")

    create = reference_create_anchors(ref)
    lyft = Config.fromfile(os.path.join(ref, STOCK[1]))
    out = {}
    for ag in lyft.target_assigner.anchor_generators:
        a = create(LYFT_FEATURE_MAP, ag["anchor_ranges"], ag["sizes"], ag["rotations"], None).reshape(-1, 7)
        idx = np.random.default_rng(0).choice(a.shape[0], 512, replace=False)
        name = ag["class_name"]
        out[name + "_sample_idx"] = idx
        out[name + "_sample"] = a[idx]
        out[name + "_checksum"] = np.array([a.astype(np.float64).sum(), (a.astype(np.float64) ** 2).sum()])
        out[name + "_shape"] = np.array(a.shape)
    np.savez_compressed(os.path.join(HERE, "anchors_lyft.npz"), **out)
    print("anchors_lyft.npz", os.path.getsize(os.path.join(HERE, "anchors_lyft.npz")), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(os.path.dirname(ROOT), "reference"))
