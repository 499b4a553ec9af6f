"""Registry shim for the reference's plugin surface (SURVEY.md §2.2).

The reference registers its classes into mmgen's ``MODELS`` / ``MODULES`` registries and builds them from
config dicts with ``build_module`` (mmgen/models/builder.py).  mmcv / mmgen are not installable offline, so this
module provides the same registries (and ``DATASETS``) and builder semantics (``type`` key, ``default_args``), and, when the real
mmgen IS importable, additionally registers every class there so the reference's own ``build_model`` finds them.
"""
import inspect


class Registry:
    def __init__(self, name):
        self.name = name
        self._module_dict = {}

    def get(self, key):
        return self._module_dict.get(key)

    def __contains__(self, key):
        return key in self._module_dict

    def register_module(self, name=None, force=False, module=None):
        def _register(cls):
            key = name or cls.__name__
            if key in self._module_dict and not force:
                raise KeyError(f'{key} is already registered in {self.name}')
            self._module_dict[key] = cls
            _mirror_to_mmgen(self.name, key, cls)
            return cls
        if module is not None:
            return _register(module)
        return _register

    def build(self, cfg, default_args=None):
        return build_from_cfg(cfg, self, default_args)


def _mirror_to_mmgen(registry_name, key, cls):
    try:   # pragma: no cover - mmgen is absent in the build container
        if registry_name == 'datasets':
            from mmgen.datasets import builder as mb
        else:
            from mmgen.models import builder as mb
        reg = getattr(mb, registry_name.upper(), None)
        if reg is not None and key not in reg.module_dict:
            reg.register_module(name=key, module=cls)
    except Exception:
        pass


def build_from_cfg(cfg, registry, default_args=None):
    """mmcv.utils.build_from_cfg semantics: cfg['type'] is a registered name or a class."""
    if not isinstance(cfg, dict) or 'type' not in cfg:
        raise KeyError(f'cfg must be a dict with a "type" key, got {cfg}')
    args = dict(cfg)
    if default_args is not None:
        for k, v in default_args.items():
            args.setdefault(k, v)
    obj_type = args.pop('type')
    if isinstance(obj_type, str):
        cls = registry.get(obj_type)
        if cls is None:
            raise KeyError(f'{obj_type} is not in the {registry.name} registry')
    elif inspect.isclass(obj_type):
        cls = obj_type
    else:
        raise TypeError(f'type must be a str or class, got {type(obj_type)}')
    return cls(**args)


MODELS = Registry('models')
MODULES = Registry('modules')
DATASETS = Registry('datasets')


def build_module(cfg, default_args=None):
    """mmgen.models.builder.build_module: look in MODULES, fall back to MODELS."""
    if isinstance(cfg, dict) and isinstance(cfg.get('type'), str) and cfg['type'] not in MODULES and cfg['type'] in MODELS:
        return build_from_cfg(cfg, MODELS, default_args)
    return build_from_cfg(cfg, MODULES, default_args)


def build_model(cfg, train_cfg=None, test_cfg=None):
    """mmgen.models.builder.build_model"""
    return build_from_cfg(cfg, MODELS, dict(train_cfg=train_cfg, test_cfg=test_cfg))


def build_dataset(cfg, default_args=None):
    """mmgen.datasets.build_dataset for a single dataset dict (ssdnerf_b200.datasets registers ShapeNetSRN)"""
    return build_from_cfg(cfg, DATASETS, default_args)
