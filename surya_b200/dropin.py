"""Drop-in binding: run the reference's *unmodified* predictors on top of the CUDA engines.

The reference has no plugin/FFI seam; a predictor reaches its network through `self.model` / `self.processor`, which
`BasePredictor.__init__` obtains from `self.model_loader_cls(checkpoint)` (surya/common/predictor.py:20-29).  The binding
therefore consists of
  * a loader class (`loader_for`) that hands out an engine model mirror and the caller's processor — the predictor
    subclass only overrides the `model_loader_cls` class attribute, every method of the reference class runs as is;
  * for recognition, `install()`: RecognitionPredictor.prefill constructs its KV cache itself from the module-level
    name `ContinuousBatchingCache` (surya/recognition/__init__.py:41-44, 391-395); that name is re-pointed at
    `SlotCache`, whose merge / trim_left / get_seq_length keep the predictor's mask bookkeeping exact while the KV data
    stays in engine slots.  No reference source file is edited.

Nothing here imports the reference at module import time: `surya` is only needed when a predictor is requested.
"""
from __future__ import annotations

import importlib
from typing import Any, Optional

from .recognition import B200SuryaModel, SlotCache


def loader_for(model: Any, processor: Any):
    """A `model_loader_cls` (surya/common/load.py ModelLoader surface: __init__(checkpoint), model(device, dtype),
    processor()) that returns pre-built objects instead of downloading a checkpoint."""

    class _Loader:
        def __init__(self, checkpoint: Optional[str] = None):
            self.checkpoint = checkpoint

        def model(self, device=None, dtype=None):
            return model

        def processor(self, device=None, dtype=None):
            return processor

    return _Loader


def install(recognition_module=None):
    """Point surya.recognition's `ContinuousBatchingCache` at SlotCache (idempotent).  Returns the module."""
    mod = recognition_module or importlib.import_module("surya.recognition")
    if getattr(mod, "ContinuousBatchingCache", None) is not SlotCache:
        mod._sb_original_cache_cls = getattr(mod, "ContinuousBatchingCache", None)
        mod.ContinuousBatchingCache = SlotCache
    return mod


def uninstall(recognition_module=None):
    mod = recognition_module or importlib.import_module("surya.recognition")
    orig = getattr(mod, "_sb_original_cache_cls", None)
    if orig is not None:
        mod.ContinuousBatchingCache = orig
        del mod._sb_original_cache_cls
    return mod


def _subclass(base, model, processor, name):
    return type(name, (base,), {"model_loader_cls": loader_for(model, processor), "__doc__": base.__doc__})


def recognition_predictor(model: B200SuryaModel, processor: Any, **kw):
    """`RecognitionPredictor` (reference class, unmodified) whose model is the engine mirror."""
    mod = install()
    return _subclass(mod.RecognitionPredictor, model, processor, "B200RecognitionPredictor")(**kw)


def detection_predictor(model: Any, processor: Any, **kw):
    """`DetectionPredictor` over B200EfficientViT (surya/detection/__init__.py:21-48, 64-132)."""
    mod = importlib.import_module("surya.detection")
    return _subclass(mod.DetectionPredictor, model, processor, "B200DetectionPredictor")(**kw)


def layout_predictor(model: Any, processor: Any, **kw):
    """`LayoutPredictor` over B200LayoutModel (surya/layout/__init__.py:24-232)."""
    mod = importlib.import_module("surya.layout")
    return _subclass(mod.LayoutPredictor, model, processor, "B200LayoutPredictor")(**kw)


def table_rec_predictor(model: Any, processor: Any, **kw):
    """`TableRecPredictor` over B200TableRecModel (surya/table_rec/__init__.py:22-331)."""
    mod = importlib.import_module("surya.table_rec")
    return _subclass(mod.TableRecPredictor, model, processor, "B200TableRecPredictor")(**kw)


def ocr_error_predictor(model: Any, processor: Any, **kw):
    """`OCRErrorPredictor` over B200DistilBert (surya/ocr_error/__init__.py:14-62); `processor` is the reference's tokenizer."""
    mod = importlib.import_module("surya.ocr_error")
    return _subclass(mod.OCRErrorPredictor, model, processor, "B200OCRErrorPredictor")(**kw)
