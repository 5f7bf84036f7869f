"""The SECOND KITTI three-class and CBGS Lyft stock configs as the reference's files parse
(tests/golden/make_golden_configs_more.py), decoded as boundary_golden.reference_config decodes the other three."""
import gzip
import json
import os

from boundary_golden import GOLDEN, decode


def reference_config_more(rel):
    from det3d.torchie import Config

    with gzip.open(os.path.join(GOLDEN, "reference_configs_more.json.gz"), "rt") as fh:
        return Config(decode(json.load(fh)[rel]), filename=None)
