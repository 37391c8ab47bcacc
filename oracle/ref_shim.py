"""Import the UNMODIFIED reference (a checkout named by $VIRTEX_REFERENCE_ROOT) -- TEST INFRASTRUCTURE ONLY.

The reference needs `albumentations` and `fvcore`, neither of which is installed here; both are irrelevant to the
model math.  This shim injects inert stand-ins into `sys.modules` (SURVEY.md section 8c) so that
`virtex.models.captioning`, `virtex.config.Config` and `virtex.factories` import and run unmodified.
Used only by `oracle/make_golden.py`; tests and the GPU path never need the reference.
"""
import ast
import os
import sys
import types

REFERENCE_ROOT = os.environ.get("VIRTEX_REFERENCE_ROOT", "")


class _CfgNode(dict):
    """Minimal stand-in for fvcore.common.config.CfgNode (yacs): attr-dict, _BASE_ files, list overrides, freeze."""
    _FROZEN = "__frozen__"

    def __init__(self, init=None):
        super().__init__()
        object.__setattr__(self, _CfgNode._FROZEN, False)
        for k, v in (init or {}).items():
            self[k] = _CfgNode(v) if isinstance(v, dict) and not isinstance(v, _CfgNode) else v

    def __getattr__(self, name):
        if name in self:
            return self[name]
        raise AttributeError(name)

    def __setattr__(self, name, value):
        if object.__getattribute__(self, _CfgNode._FROZEN):
            raise AttributeError(f"Attempted to set {name} on an immutable CfgNode")
        self[name] = value

    def freeze(self):
        object.__setattr__(self, _CfgNode._FROZEN, True)
        for v in self.values():
            if isinstance(v, _CfgNode):
                v.freeze()

    def clone(self):
        import copy
        return copy.deepcopy(self)

    @staticmethod
    def _load_yaml(path):
        import yaml
        with open(path) as f:
            cfg = yaml.safe_load(f) or {}
        base = cfg.pop("_BASE_", None)
        if base is not None:
            if not os.path.isabs(base):
                base = os.path.join(os.path.dirname(path), base)
            merged = _CfgNode._load_yaml(base)
            _CfgNode._merge(cfg, merged)
            return merged
        return cfg

    @staticmethod
    def _merge(src, dst):
        for k, v in src.items():
            if isinstance(v, dict) and isinstance(dst.get(k), dict):
                _CfgNode._merge(v, dst[k])
            else:
                dst[k] = _CfgNode(v) if isinstance(v, dict) and isinstance(dst, _CfgNode) else v

    def merge_from_file(self, path):
        _CfgNode._merge(_CfgNode._load_yaml(path), self)

    def merge_from_list(self, lst):
        assert len(lst) % 2 == 0
        for key, value in zip(lst[0::2], lst[1::2]):
            node = self
            parts = key.split(".")
            for p in parts[:-1]:
                node = node[p]
            if isinstance(value, str):
                try:
                    value = ast.literal_eval(value)
                except (ValueError, SyntaxError):
                    pass
            dict.__setitem__(node, parts[-1], value)

    def dump(self, **kw):
        import yaml

        def plain(n):
            return {k: plain(v) if isinstance(v, dict) else v for k, v in n.items()}
        return yaml.safe_dump(plain(self), **kw)


def install():
    """Make `import virtex` resolve to the reference tree with stubbed third-party deps."""
    if not available():
        raise RuntimeError("set VIRTEX_REFERENCE_ROOT to a checkout of the reference (kdexd/virtex)")
    if "albumentations" not in sys.modules:
        alb = types.ModuleType("albumentations")

        class BasicTransform:  # noqa: D401
            def __init__(self, *a, **k):
                pass

        for n in ("BasicTransform", "RandomResizedCrop", "CenterCrop", "Resize", "SmallestMaxSize", "Normalize",
                  "Compose", "ColorJitter", "HorizontalFlip", "ImageOnlyTransform"):
            setattr(alb, n, type(n, (BasicTransform,), {}))
        alb.BasicTransform = BasicTransform
        sys.modules["albumentations"] = alb
    if "fvcore" not in sys.modules:
        fv = types.ModuleType("fvcore")
        fvc = types.ModuleType("fvcore.common")
        fvcc = types.ModuleType("fvcore.common.config")
        fvcc.CfgNode = _CfgNode
        fvcd = types.ModuleType("fvcore.common.download")
        fvcd.download = lambda *a, **k: (_ for _ in ()).throw(RuntimeError("no network"))
        fv.common, fvc.config, fvc.download = fvc, fvcc, fvcd
        sys.modules.update({"fvcore": fv, "fvcore.common": fvc, "fvcore.common.config": fvcc,
                            "fvcore.common.download": fvcd})
    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)


def available():
    """True when $VIRTEX_REFERENCE_ROOT names a reference checkout OUTSIDE this repository (this repository's own
    `virtex/` alias package must never stand in for the reference)."""
    if not REFERENCE_ROOT:
        return False
    root = os.path.realpath(REFERENCE_ROOT)
    here = os.path.realpath(os.path.join(os.path.dirname(os.path.abspath(__file__)), os.pardir))
    if root == here or root.startswith(here + os.sep):
        raise RuntimeError(f"VIRTEX_REFERENCE_ROOT={REFERENCE_ROOT} lies inside this repository, not in a reference checkout")
    return os.path.isdir(os.path.join(root, "virtex"))
