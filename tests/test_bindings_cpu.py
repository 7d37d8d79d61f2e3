"""CPU: every ctypes declaration of the Python front end (_lib.lib() and trainer._bind()) has as many argument types as its declaration in
include/psb200.h has parameters, so a list that drifts from the header fails here instead of passing garbage to the library."""
import os
import re

from photo_slam_b200 import _lib, trainer

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "psb200.h")


def _header_arity():
    """name -> number of parameters of every psb_* function declared in the header (`(void)` has none)."""
    txt = re.sub(r"/\*.*?\*/|//[^\n]*", "", open(HEADER).read(), flags=re.S)
    arity = {}
    for name, params in re.findall(r"\b(psb_[a-z0-9_]+)\s*\(([^()]*)\)\s*;", txt):
        params = params.strip()
        arity[name] = 0 if params in ("", "void") else params.count(",") + 1
    return arity


def test_header_parse_finds_every_exported_function():
    assert set(_header_arity()) == set(_lib.exported_symbols())


def test_every_declared_argtypes_matches_the_header():
    L = trainer._bind()
    arity = _header_arity()
    declared = {name: getattr(L, name).argtypes for name in arity if getattr(L, name).argtypes is not None}
    # everything the trainer, data-parallel, densification and debug families call is declared
    for name in arity:
        if name.startswith(("psb_trainer_", "psb_dp_", "psb_adam_", "psb_densify_", "psb_prune_", "psb_rasterize_", "psb_debug_")):
            assert name in declared, name
    bad = {name: (len(args), arity[name]) for name, args in declared.items() if len(args) != arity[name]}
    assert not bad, bad
