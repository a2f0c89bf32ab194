"""Drop-in alias: `from isdf.modules import trainer` (reference train.py:16) resolves to isdf_b200.

Put this repo's root on sys.path BEFORE the reference checkout and the reference drivers
(isdf/train/train.py, train_vis.py, batch_train) import this implementation unchanged:

* `isdf.modules`, `isdf.geometry`, `isdf.datasets`, `isdf.eval` are this repo's packages;
* every other sub-package the drivers import (`isdf.visualisation`, `isdf.train`, `isdf.ros_utils`, ...) and
  every sub-module this repo does not provide (`isdf.eval.plot_utils`, `isdf.datasets.sdf_util`, ...) is taken
  from the reference checkout found later on sys.path -- a regular package shadows the reference's namespace
  package, so its directory is appended to the package search paths here;
* a name a mirrored module does not define (e.g. `isdf.geometry.transform.to_trimesh`) falls back to the
  reference's module of the same name, loaded lazily under `isdf_reference.*`.
"""
import importlib.util
import os
import sys
import warnings

import isdf_b200
from isdf_b200 import modules, geometry, datasets, eval  # noqa: F401,A004

_HERE = os.path.dirname(os.path.abspath(__file__))


def _find_reference():
    for entry in sys.path:
        cand = os.path.join(os.path.abspath(entry or "."), "isdf")
        if os.path.abspath(cand) != _HERE and os.path.isfile(os.path.join(cand, "modules", "trainer.py")):
            return cand
    return None


_REF = _find_reference()


def _fallback_getattr(mod, ref_file):
    """Module-level __getattr__: names this repo's module lacks come from the reference's file."""
    state = {}

    def __getattr__(name):
        if name.startswith("__"):
            raise AttributeError(name)
        if "ref" not in state:
            spec = importlib.util.spec_from_file_location("isdf_reference." + mod.__name__.split(".", 1)[1], ref_file)
            ref = importlib.util.module_from_spec(spec)
            spec.loader.exec_module(ref)
            state["ref"] = ref
        try:
            val = getattr(state["ref"], name)
        except AttributeError:
            raise AttributeError("module %r has no attribute %r (nor has the reference's %s)" % (mod.__name__, name, ref_file))
        if name not in state.setdefault("warned", set()):
            # never silent: a name of a mirrored (hot-path) module that is served by the reference's Python code is worth
            # knowing about -- it is either out-of-scope tooling (to_trimesh, plotting helpers) or a gap in this package
            state["warned"].add(name)
            warnings.warn("isdf_b200: %s.%s is not provided by this implementation; using the reference's %s"
                          % (mod.__name__, name, ref_file), stacklevel=2)
        return val
    return __getattr__


for _name, _mod in (("modules", modules), ("geometry", geometry), ("datasets", datasets), ("eval", eval)):
    sys.modules["isdf." + _name] = _mod
    for _sub in dir(_mod):
        _obj = getattr(_mod, _sub)
        if getattr(_obj, "__name__", "").startswith("isdf_b200." + _name + "."):
            sys.modules["isdf.%s.%s" % (_name, _sub)] = _obj
            if _REF:
                _ref_file = os.path.join(_REF, _name, _sub + ".py")
                if os.path.isfile(_ref_file) and not hasattr(_obj, "__getattr__"):
                    _obj.__getattr__ = _fallback_getattr(_obj, _ref_file)
    if _REF and os.path.isdir(os.path.join(_REF, _name)):
        _mod.__path__.append(os.path.join(_REF, _name))          # sub-modules this repo does not provide
if _REF:
    __path__.append(_REF)                                          # isdf.visualisation, isdf.train, ...
__version__ = isdf_b200.__version__
