"""Alias package: ``import cleandiffuser`` resolves to ``cleandiffuser_b200`` (use when the reference is NOT installed).

Put ``<repo>/compat`` (and the repo root) on PYTHONPATH; the reference's pipeline scripts then import
``cleandiffuser.diffusion`` / ``nn_diffusion`` / ``nn_condition`` / ``utils`` unchanged and get the H100 engine.
Sub-packages outside the hot path (dataset, env, classifier, invdynamic ...) are deliberately absent."""
import importlib
import sys

import cleandiffuser_b200 as _impl

for _name in ("diffusion", "nn_diffusion", "nn_condition", "utils"):
    _mod = importlib.import_module(f"cleandiffuser_b200.{_name}")
    sys.modules[f"{__name__}.{_name}"] = _mod
    globals()[_name] = _mod

__version__ = _impl.__version__
__cleandiffuser_b200_alias__ = True

# sub-packages of the reference that are NOT on the hot path and are not provided by the alias
_NOT_PORTED = ("classifier", "nn_classifier", "dataset", "env", "invdynamic")


def __getattr__(name):
    if name in _NOT_PORTED:
        raise ImportError(f"cleandiffuser.{name} is outside the H100 engine's scope (SURVEY section 8) and not part of the alias "
                          "package: install the reference and call cleandiffuser_b200.install() instead (drop-in route A)")
    raise AttributeError(name)
