import os, sys
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100: -m gpu)")
    config.addinivalue_line("markers", "ref: needs oracle/_ref (the compiled reference); skipped when absent")


# Fuzzing aid (tools/fuzz_oracle.py): every test draws its inputs from np.random.default_rng(<constant>); THOR_FUZZ_OFFSET=k shifts all
# those constants, turning the fixed pins into fresh random cases.  Unset (the default, and what the driver runs): no effect.
_FUZZ = int(os.environ.get("THOR_FUZZ_OFFSET", "0") or 0)
if _FUZZ:
    import numpy as _np
    _orig_rng = _np.random.default_rng
    _np.random.default_rng = lambda seed=None: _orig_rng(None if seed is None else int(seed) + 1000003 * _FUZZ)
