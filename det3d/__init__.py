"""`det3d` import-path alias of det3d_b200.

Det3D configs and user code import `det3d.builder`, `det3d.utils.config_tool`,
`det3d.models...`, `det3d.core.input.voxel_generator`, ... (e.g.
examples/second/configs/kitti_car_vfev3_spmiddlefhd_rpn1_mghead_syncbn.py:4-5).  This
package makes every `det3d.<path>` resolve to the SAME module object as
`det3d_b200.<path>`, so those imports work unchanged against the H100-native
implementation.
"""
import importlib
import importlib.abc
import importlib.util
import sys

import det3d_b200 as _impl

_PREFIX = __name__ + "."
_TARGET = _impl.__name__ + "."


class _AliasLoader(importlib.abc.Loader):
    def __init__(self, target):
        self._target = target

    def create_module(self, spec):
        return importlib.import_module(self._target)

    def exec_module(self, module):
        pass


class _AliasFinder(importlib.abc.MetaPathFinder):
    def find_spec(self, fullname, path=None, target=None):
        if not fullname.startswith(_PREFIX):
            return None
        real = _TARGET + fullname[len(_PREFIX):]
        try:
            if importlib.util.find_spec(real) is None:
                return None
        except ModuleNotFoundError:
            return None
        return importlib.util.spec_from_loader(fullname, _AliasLoader(real))


if not any(isinstance(f, _AliasFinder) for f in sys.meta_path):
    sys.meta_path.insert(0, _AliasFinder())

__version__ = _impl.__version__
__path__ = []  # a package with no files of its own: submodules come from the finder


def __getattr__(name):
    # det3d.torchie / det3d.models / ... as attributes
    try:
        return importlib.import_module(_PREFIX + name)
    except ModuleNotFoundError as e:
        raise AttributeError(name) from e
