"""Golden config of the nuScenes PointPillars stock config, produced by the REFERENCE's own file.

Run with a Det3D reference checkout (V2AI/Det3D @ 230bb199) at REF (default ../reference beside the repository, or
the first argument):

    python tests/golden/make_golden_pillars_nusc.py [REF]

* reference_config_pillars_nusc.json.gz -- examples/point_pillars/configs/nusc_all_point_pillars_mghead_syncbn.py as
  `Config.fromfile` parses it, encoded by make_golden_boundary.encode (the encoding of reference_configs.json.gz).  A
  file of its own, so that the existing fixtures stay byte-identical; the gzip header carries no timestamp.
"""
import gzip
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)

from make_golden_boundary import encode  # noqa: E402  (also puts the repository root on sys.path)

REL = "examples/point_pillars/configs/nusc_all_point_pillars_mghead_syncbn.py"
OUT = "reference_config_pillars_nusc.json.gz"


def main(ref):
    from det3d.torchie import Config

    cfg = Config.fromfile(os.path.join(ref, REL))
    data = {REL: {k: encode(cfg[k]) for k in cfg}}
    with open(os.path.join(HERE, OUT), "wb") as raw, gzip.GzipFile(filename="", mode="wb", fileobj=raw, mtime=0) as gz:
        gz.write(json.dumps(data, sort_keys=True).encode())
    print(OUT, os.path.getsize(os.path.join(HERE, OUT)), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(os.path.dirname(ROOT), "reference"))
