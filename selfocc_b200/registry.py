"""Registry shim: the reference finds its modules by ``type=`` strings through mmengine/mmseg
registries (SURVEY.md 8b: ``@MODELS.register_module()``, ``HEADS``, ``build_head`` ...).  When
mmengine/mmseg are importable the classes of this package register into THOSE registries (so
``train.py`` / ``eval_*.py`` pick them up unchanged); otherwise a self-contained registry with the
same surface (``register_module``, ``build``, ``get``) is used.
"""
import copy
import inspect


class Registry:
    def __init__(self, name):
        self.name = name
        self._modules = {}

    def register_module(self, name=None, force=False, module=None):
        def _reg(cls):
            key = name or cls.__name__
            if key in self._modules and not force:
                raise KeyError('%s is already registered in %s' % (key, self.name))
            self._modules[key] = cls
            return cls
        return _reg(module) if module is not None else _reg

    def get(self, key):
        return self._modules.get(key)

    def __contains__(self, key):
        return key in self._modules

    def build(self, cfg, **default_args):
        if cfg is None:
            return None
        if not isinstance(cfg, dict) or 'type' not in cfg:
            raise TypeError('cfg must be a dict with a "type" key, got %r' % (cfg,))
        args = copy.deepcopy(dict(cfg))
        for k, v in default_args.items():
            args.setdefault(k, v)
        t = args.pop('type')
        cls = self.get(t) if isinstance(t, str) else t
        if cls is None:
            raise KeyError('%s is not in the %s registry' % (t, self.name))
        if not inspect.isclass(cls):
            raise TypeError('type must be a str or class')
        return cls(**args)


try:  # pragma: no cover - mmengine is absent in the build container
    from mmengine.registry import MODELS as _MM_MODELS
    try:
        from mmseg.registry import MODELS as _SEG_MODELS
    except Exception:
        _SEG_MODELS = _MM_MODELS
    MODELS = _SEG_MODELS
    HEADS = _SEG_MODELS
    HAVE_MMENGINE = True
except Exception:
    MODELS = Registry('selfocc_b200.models')
    HEADS = MODELS  # mmseg>=1.0 aliases HEADS to MODELS as well
    HAVE_MMENGINE = False


# The reference's loss registry is private to its `loss` package (loss/__init__.py: OPENOCC_LOSS = Registry('openocc_loss')),
# so this package cannot register into it at import time; its losses live here and INTEGRATION.md shows the two
# `OPENOCC_LOSS.register_module(module=..., force=True)` lines that hand them to the reference's MultiLoss.
LOSSES = Registry('selfocc_b200.losses')


def build_head(cfg):
    """mmseg.models.builder.build_head: the reference builds lifter, encoder AND head with it
    (model/segmentor/base_segmentor.py:27-32)."""
    return MODELS.build(cfg)


build_attention = build_positional_encoding = build_transformer_layer = build_feedforward_network = build_head
