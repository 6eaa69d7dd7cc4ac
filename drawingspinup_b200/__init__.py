"""drawingspinup_b200 - CUDA (H100, sm_90a) engine for DrawingSpinUp's per-frame stylization hot path.

Public surface (mirrors ``3_style_translator/training/models.py`` for the inference path):

* :class:`GeneratorJ_RIC`, :class:`GeneratorJ` - drop-in classes for ``training.models``.
* :func:`install` - rebind those two names inside the reference's ``training.models`` so that
  ``training.trainers.build_model`` (trainers.py:33-35) builds the CUDA engine.
* :mod:`drawingspinup_b200.pipeline` - device-resident stage-1 -> stage-2 frame pipeline with
  frame sharding across GPUs; :mod:`drawingspinup_b200.run` - launcher for the unmodified
  ``test_stage1.py`` / ``test_stage2.py``.
"""
from .models import GeneratorJ, GeneratorJ_RIC, ric_offsets  # noqa: F401

__all__ = ["GeneratorJ", "GeneratorJ_RIC", "ric_offsets", "install", "uninstall"]


def install(models_module=None):
    """Rebind ``GeneratorJ_RIC`` / ``GeneratorJ`` in the reference's ``training.models`` module.

    ``build_model`` resolves the class by name at call time (``getattr(m, model_type)``,
    trainers.py:33-35), so after this call the unmodified reference scripts construct, load and
    call the CUDA engine.  Returns the patched module."""
    if models_module is None:
        import importlib
        models_module = importlib.import_module("training.models")
    # the reference classes call ``super(GeneratorJ_RIC, self).__init__()`` through the module-level NAME (models.py:204),
    # so they cannot be constructed while the names are rebound: build reference models (in-process A/B checks) before
    # install() or after uninstall().  The originals stay reachable as ``_dsu_original``.
    if not hasattr(models_module, "_dsu_original"):
        models_module._dsu_original = {"GeneratorJ_RIC": getattr(models_module, "GeneratorJ_RIC", None),
                                       "GeneratorJ": getattr(models_module, "GeneratorJ", None)}
    models_module.GeneratorJ_RIC = GeneratorJ_RIC
    models_module.GeneratorJ = GeneratorJ
    return models_module


def uninstall(models_module=None):
    """Undo :func:`install`: restore the reference's own ``GeneratorJ_RIC`` / ``GeneratorJ`` classes."""
    if models_module is None:
        import importlib
        models_module = importlib.import_module("training.models")
    orig = getattr(models_module, "_dsu_original", None)
    if orig:
        for name, cls in orig.items():
            if cls is not None:
                setattr(models_module, name, cls)
        del models_module._dsu_original
    return models_module
