"""Minimal stand-in for ``mmcv.Config.fromfile`` so the reference's python-dict configs load unchanged
(tools/test.py:118-120): executes the file, follows ``_base_`` inheritance with dict merging (``_delete_`` honoured)
and supports ``--cfg-options`` style dotted overrides.  If mmcv is importable, the real Config is used instead."""
import os
import runpy


class ConfigDict(dict):
    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e

    def __setattr__(self, k, v):
        self[k] = v


def _wrap(x):
    if isinstance(x, dict):
        return ConfigDict({k: _wrap(v) for k, v in x.items()})
    if isinstance(x, (list, tuple)):
        return type(x)(_wrap(v) for v in x)
    return x


def _plain(x):
    if isinstance(x, dict):
        return {k: _plain(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return type(x)(_plain(v) for v in x)
    if isinstance(x, range):
        return list(x)
    return x


def _merge(base, new):
    out = dict(base)
    for k, v in new.items():
        if isinstance(v, dict) and isinstance(out.get(k), dict) and not v.get('_delete_', False):
            out[k] = _merge(out[k], v)
        else:
            out[k] = {kk: vv for kk, vv in v.items() if kk != '_delete_'} if isinstance(v, dict) else v
    return out


def _load(path):
    ns = runpy.run_path(path)
    cfg = {k: v for k, v in ns.items() if not k.startswith('__') and not callable(v) and not isinstance(v, type(os))}
    base = cfg.pop('_base_', None)
    if base is not None:
        bases = [base] if isinstance(base, str) else list(base)
        merged = {}
        for b in bases:
            merged = _merge(merged, _load(os.path.join(os.path.dirname(path), b)))
        cfg = _merge(merged, cfg)
    return cfg


class Config:
    @staticmethod
    def fromfile(filename):
        try:   # pragma: no cover
            from mmcv import Config as _C
            return _C.fromfile(filename)
        except ImportError:
            return _wrap(_load(os.path.abspath(filename)))

    @staticmethod
    def dump(cfg, filename):
        """writes `cfg` as a python config file, one `name = value` line per top-level key, that `fromfile` reads back to an equal
        dict (values must be plain python literals: dicts, lists, tuples, strings, numbers, booleans, None)"""
        with open(filename, 'w') as f:
            for k, v in cfg.items():
                f.write(f'{k} = {_plain(v)!r}\n')

    @staticmethod
    def merge_options(cfg, options):
        """`--cfg-options a.b.c=v` semantics on a loaded config"""
        for key, value in options.items():
            d = cfg
            parts = key.split('.')
            for p in parts[:-1]:
                d = d.setdefault(p, ConfigDict())
            d[parts[-1]] = _wrap(value)
        return cfg
