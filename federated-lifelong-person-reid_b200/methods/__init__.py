"""Method registry keyed by the reference's strings (``methods/__init__.py:3-14``). Every entry is a module that
exports ``Operator``, ``Client``, ``Server`` and optionally ``Model``."""
import importlib

_NAMES = {
    "baseline": "baseline",
    "ewc": "ewc",
    "mas": "mas",
    "si": "si",
    "icarl": "icarl",
    "fedavg": "fedavg",
    "fedprox": "fedprox",
    "fedcurv": "fedcurv",
    "fedweit": "fedweit",
    "fedstil": "fedstil",
    "fedstil-atten": "fedstil_atten",
}


class _Registry(dict):
    def __missing__(self, key):
        if key not in _NAMES:
            raise KeyError(f"unknown method '{key}' (known: {sorted(_NAMES)})")
        mod = importlib.import_module(f"{__name__}.{_NAMES[key]}")
        self[key] = mod
        return mod

    def keys(self):
        return _NAMES.keys()

    def __contains__(self, key):
        return key in _NAMES

    def __iter__(self):
        return iter(_NAMES)


methods = _Registry()
