"""Make the reference's own scripts pick up the H100 implementation without editing them.

    import esr_b200.dropin; esr_b200.dropin.install()        # before `from models.model import *`

install() registers, under the module names the reference imports (SURVEY.md 8b):
  `_ext`                                          -> esr_b200.dcn_v2_ext      (models/DCNv2/dcn_v2.py:13)
  `dataloader.cython_cnt2event.cnt2event`          -> esr_b200.cnt2event       (cnt2event_api.py:1)
  `dataloader.cython_event_redistribute.event_redistribute` -> esr_b200.event_redistribute (encodings.py:5)
  `models.model` : a module exposing DeepRecurrNet  -> esr_b200.model          (train_ours_cnt_seq.py:20, infer_ours_cnt.py:14)
and, optionally (patch_encodings=True), replaces the hot functions of an already imported `dataloader.encodings`, and
(patch_loader=True) registers `dataloader.h5dataloader` exposing esr_b200.loader.HDF5DataLoaderSequence and an
HDF5DataLoader that raises ESRError when constructed (train_ours_cnt_seq.py:18 imports both names; the per-frame
H5Dataset loader is not served).
"""
import importlib.util
import sys
import types


def _package(name):
    """The package a replaced leaf module lives in.  When the reference checkout is on sys.path the REAL (namespace) package
    is used, so that its other modules (cnt2event_api.py, ...) stay importable next to the replaced leaf; otherwise a stub."""
    if name in sys.modules:
        return sys.modules[name]
    try:
        if importlib.util.find_spec(name) is not None:
            return importlib.import_module(name)
    except (ImportError, ValueError, AttributeError):
        pass
    parent, _, leaf = name.rpartition(".")
    m = types.ModuleType(name)
    m.__path__ = []                                    # a package, with nothing else inside
    sys.modules[name] = m
    if parent:
        setattr(_package(parent), leaf, m)
    return m


def install(patch_models=True, patch_encodings=False, patch_loader=False):
    from . import cnt2event, dcn_v2_ext, event_redistribute, model
    sys.modules["_ext"] = dcn_v2_ext
    _package("dataloader.cython_cnt2event").cnt2event = cnt2event
    sys.modules["dataloader.cython_cnt2event.cnt2event"] = cnt2event
    _package("dataloader.cython_event_redistribute").event_redistribute = event_redistribute
    sys.modules["dataloader.cython_event_redistribute.event_redistribute"] = event_redistribute
    if patch_models:
        m = types.ModuleType("models.model")
        m.DeepRecurrNet = model.DeepRecurrNet
        m.__all__ = ["DeepRecurrNet"]
        sys.modules["models.model"] = m
        try:
            _package("models").model = m
        except Exception:
            pass
    if patch_encodings and "dataloader.encodings" in sys.modules:
        from . import encodings
        ref = sys.modules["dataloader.encodings"]
        for name in ("events_to_image", "events_to_channels", "cython_event_redistribute", "multiprocess_cython", "stack2cnt"):
            setattr(ref, name, getattr(encodings, name))
    if patch_loader:
        from . import loader
        m = types.ModuleType("dataloader.h5dataloader")
        m.HDF5DataLoaderSequence = loader.HDF5DataLoaderSequence
        m.HDF5DataLoader = _HDF5DataLoader
        sys.modules["dataloader.h5dataloader"] = m
        _package("dataloader").h5dataloader = m


class _HDF5DataLoader:
    """dataloader/h5dataloader.py:HDF5DataLoader (one H5Dataset item per batch entry) is not served: constructing it raises."""

    def __init__(self, *args, **kwargs):
        from ._lib import ESRError
        raise ESRError("HDF5DataLoader (per-frame H5Dataset batches) is not implemented; train from "
                       "HDF5DataLoaderSequence (esr_b200.loader)")
