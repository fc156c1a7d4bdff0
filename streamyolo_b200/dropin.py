"""Make ``from exps.model.yolox import YOLOX`` (what the reference's cfgs/*.py do,
/root/reference/cfgs/s_s50_onex_dfp_tal_flip.py:35-37) resolve to this implementation.

    import streamyolo_b200.dropin; streamyolo_b200.dropin.install()     # before get_exp(...)

Registers ``exps``, ``exps.model`` and the five model modules (yolox, dfp_pafpn, darknet, tal_head, pipe_head) in ``sys.modules`` (existing ``exps`` packages are
kept: only the ``exps.model.*`` names are redirected)."""
import importlib
import sys
import types

_NAMES = ("yolox", "dfp_pafpn", "darknet", "tal_head", "pipe_head")      # every module of the reference's exps/model/


def install(postprocess: bool = True) -> None:
    """``postprocess=True`` also points ``yolox.utils.postprocess`` (imported by the reference's evaluators,
    exps/evaluators/onex_stream_evaluator.py:14,148) at the device NMS when the yolox package is importable."""
    pkg = importlib.import_module("streamyolo_b200.model")
    if "exps" not in sys.modules:
        root = types.ModuleType("exps")
        root.__path__ = []
        sys.modules["exps"] = root
    sys.modules["exps.model"] = pkg
    setattr(sys.modules["exps"], "model", pkg)
    for n in _NAMES:
        sys.modules[f"exps.model.{n}"] = importlib.import_module(f"streamyolo_b200.model.{n}")
    if postprocess:
        try:
            import yolox.utils as yu                                    # absent in the build image; present in a real checkout
            from .postprocess import postprocess as device_postprocess
            yu.postprocess = device_postprocess
            if hasattr(yu, "boxes"):
                yu.boxes.postprocess = device_postprocess
        except ImportError:
            pass
