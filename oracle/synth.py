"""Compatibility alias: the seeded synthetic inputs / weights live in ``synthdata.py`` at the repo root (they contain
no reference arithmetic, and bench.py's GPU arm needs them without touching ``oracle/``).  The tests and the oracle
keep importing ``oracle.synth``."""
from synthdata import *  # noqa: F401,F403
from synthdata import _bilinear_zero, _blur_filt, _bn, _conv, _head_state, _texture  # noqa: F401
