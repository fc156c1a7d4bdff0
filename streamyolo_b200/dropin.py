"""Make ``from exps.model.yolox import YOLOX`` (what the reference's cfgs/*.py do,
/root/reference/cfgs/s_s50_onex_dfp_tal_flip.py:35-37) resolve to this implementation.

    import streamyolo_b200.dropin; streamyolo_b200.dropin.install()     # before get_exp(...)

Registers ``exps.model`` and the five model modules (yolox, dfp_pafpn, darknet, tal_head, pipe_head) in ``sys.modules``.
An ``exps`` package that is importable (the reference checkout's, when ``tools/train.py`` runs from its root) is imported
and kept, so that ``exps.train_utils`` and ``exps.evaluators`` stay its own; only the ``exps.model.*`` names are
redirected.  Without one, an empty ``exps`` package is registered."""
import importlib
import importlib.util
import sys
import types

_NAMES = ("yolox", "dfp_pafpn", "darknet", "tal_head", "pipe_head")      # every module of the reference's exps/model/


_EVALUATORS = (("onex_stream_evaluator", "ONEX_COCOEvaluator", "onex"), ("twox_stream_evaluator", "TWOX_COCOEvaluator", "twox"),
               ("still_stream_evaluator", "STILL_COCOEvaluator", "still"))


def install(postprocess: bool = True, evaluators: bool = False, trainer: bool = False, virtual_ranks: int = 1) -> None:
    """``postprocess=True`` also points ``yolox.utils.postprocess`` (imported by the reference's evaluators,
    exps/evaluators/onex_stream_evaluator.py:14,148) at the device NMS when the yolox package is importable.

    ``evaluators=True`` replaces ``ONEX_COCOEvaluator``, ``TWOX_COCOEvaluator`` and ``STILL_COCOEvaluator`` in their
    ``exps.evaluators.*`` modules by subclasses whose ``evaluate`` runs the batch loop on the device
    (``streamyolo_b200.evaluate``); ``evaluate_prediction`` (COCOeval, per-class AP) stays the reference's.  Nothing
    happens when the reference's evaluators, yolox or pycocotools cannot be imported.

    ``trainer=True`` replaces ``exps.train_utils.double_trainer.Trainer`` (what every shipped cfg's ``get_trainer``
    imports) by a subclass whose loop runs on the device (``streamyolo_b200.train_loop``): JPEG files in, one CUDA graph
    replay per iteration.  Nothing happens when that module or yolox cannot be imported.  ``install(trainer=True,
    evaluators=True)`` is the recommended pair for ``tools/train.py``: the per-epoch evaluation then runs on the device too.
    ``virtual_ranks=K`` (with ``trainer=True``): every process runs K ranks of a W x K-rank run one after another, so
    ``tools/train.py -d 1 -b 32`` with K = 8 trains as the README's ``-d 8 -b 32`` does (``train_loop.DeviceTrainer``)."""
    pkg = importlib.import_module("streamyolo_b200.model")
    if "exps" not in sys.modules:
        if importlib.util.find_spec("exps") is not None:   # the reference checkout's own package: its exps.train_utils,
            importlib.import_module("exps")                 # exps.evaluators, ... must stay importable
        else:
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
    if evaluators:
        install_evaluators()
    if trainer:
        install_trainer(virtual_ranks)


def install_evaluators() -> None:
    """The ``evaluators=True`` part of ``install``."""
    try:
        import pycocotools  # noqa: F401
        import yolox.utils  # noqa: F401
    except ImportError:
        return
    from .evaluate import DeviceEvaluator, device_evaluator
    for mod, name, rule in _EVALUATORS:
        try:
            m = importlib.import_module(f"exps.evaluators.{mod}")
        except ImportError:
            continue
        base = getattr(m, name, None)
        if base is not None and not issubclass(base, DeviceEvaluator):
            setattr(m, name, device_evaluator(base, rule))


def install_trainer(virtual_ranks: int = 1) -> None:
    """The ``trainer=True`` part of ``install``; a second call only sets ``virtual_ranks``."""
    if int(virtual_ranks) != virtual_ranks or virtual_ranks < 1:
        raise ValueError(f"install: virtual_ranks must be a positive integer, got {virtual_ranks!r}")
    try:
        import yolox  # noqa: F401
        m = importlib.import_module("exps.train_utils.double_trainer")
    except ImportError:
        return
    from .train_loop import DeviceTrainer, device_trainer
    base = getattr(m, "Trainer", None)
    if base is not None and not issubclass(base, DeviceTrainer):
        m.Trainer = device_trainer(base)
    if base is not None:
        m.Trainer.virtual_ranks = int(virtual_ranks)
