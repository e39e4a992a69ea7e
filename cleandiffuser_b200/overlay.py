"""Drop-in route A ("overlay"): keep the reference installed and let its scripts run unchanged on this engine.

``install()`` rebinds the hot-path classes INSIDE the imported reference package,

    cleandiffuser.diffusion.{DiscreteDiffusionSDE, ContinuousDiffusionSDE, ContinuousConsistencyModel, ContinuousEDM}
    (+ the defining sub-modules cleandiffuser.diffusion.diffusionsde / .consistency_model / .newedm)

to this package's classes, so that a pipeline's ``from cleandiffuser.diffusion import DiscreteDiffusionSDE`` -- and
everything else it imports from the reference: datasets, envs, classifiers, ``nn_classifier``, ``utils.report_parameters``
... -- keeps working, while ``agent.sample(...)`` runs the reverse loop on the sm_90a engine.  The reference's own
``nn_diffusion`` / ``nn_condition`` modules are accepted as they are: the lowering recognises backbones structurally
(class name + attributes, ``engine/lower.py``), and the PyTorch path calls them like the reference does.

    import cleandiffuser_b200; cleandiffuser_b200.install()          # first line of a script, or
    python -m cleandiffuser_b200.run pipelines/diffuser_d4rl_mujoco.py mode=inference ...   # script untouched

Reference surfaces mirrored: cleandiffuser/diffusion/__init__.py:1-5, diffusionsde.py:247,609, consistency_model.py:58.
"""
import importlib
import sys
from typing import Dict, List, Tuple

_PATCHED: List[Tuple[object, str, object]] = []      # (module, attribute, original)

# reference module -> names rebound there
_TARGETS: Dict[str, Tuple[str, ...]] = {
    "cleandiffuser.diffusion": ("DiscreteDiffusionSDE", "ContinuousDiffusionSDE", "ContinuousConsistencyModel", "ContinuousEDM",
                                "DiscreteRectifiedFlow", "ContinuousRectifiedFlow"),
    "cleandiffuser.diffusion.newedm": ("ContinuousEDM",),
    "cleandiffuser.diffusion.ddpm": ("DDPM",),
    "cleandiffuser.diffusion.edm": ("EDM",),
    "cleandiffuser.diffusion.rectifiedflow": ("DiscreteRectifiedFlow", "ContinuousRectifiedFlow"),
    "cleandiffuser.diffusion.diffusionsde": ("DiscreteDiffusionSDE", "ContinuousDiffusionSDE"),
    "cleandiffuser.diffusion.consistency_model": ("ContinuousConsistencyModel",),
}


def reference_available() -> bool:
    """Is the real reference package importable (and not this repo's ``compat/`` alias)?"""
    try:
        mod = importlib.import_module("cleandiffuser")
    except Exception:
        return False
    return not getattr(mod, "__cleandiffuser_b200_alias__", False)


def install(strict: bool = True) -> List[str]:
    """Rebind the reference's sampler classes to the H100 engine's.  Returns the patched ``module.attr`` names.
    ``strict=False`` returns [] instead of raising when the reference is not importable.  Idempotent."""
    from . import diffusion as ours
    if _PATCHED:
        return [f"{m.__name__}.{a}" for m, a, _ in _PATCHED]
    if not reference_available():
        if strict:
            raise ImportError("cleandiffuser_b200.install(): the reference package `cleandiffuser` is not importable "
                              "(install it, or use the alias package under compat/ instead)")
        return []
    done = []
    for mod_name, names in _TARGETS.items():
        try:
            mod = importlib.import_module(mod_name)
        except Exception:
            if strict:
                raise
            continue
        for name in names:
            if hasattr(mod, name) and hasattr(ours, name):
                _PATCHED.append((mod, name, getattr(mod, name)))
                setattr(mod, name, getattr(ours, name))
                done.append(f"{mod_name}.{name}")
    return done


def uninstall() -> None:
    """Undo ``install()``."""
    while _PATCHED:
        mod, name, orig = _PATCHED.pop()
        setattr(mod, name, orig)


def installed() -> bool:
    return bool(_PATCHED)


def main(argv=None) -> None:
    """``python -m cleandiffuser_b200.run <script.py> [args...]``: install the overlay, then run the script as __main__."""
    import runpy
    argv = list(sys.argv[1:] if argv is None else argv)
    if not argv:
        raise SystemExit("usage: python -m cleandiffuser_b200.run <script.py> [script args...]")
    install(strict=True)
    sys.argv = argv
    runpy.run_path(argv[0], run_name="__main__")
