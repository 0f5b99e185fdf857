"""CPU-side checks of include/adanerf_b200_views.h: the library exports every symbol the header declares, the ctypes shim
binds exactly those, and the single-view header declares none of them."""
import ctypes
import os
import re

from conftest import ROOT


def _declared(name):
    with open(os.path.join(ROOT, "include", name)) as fh:
        return set(re.findall(r"\b(adn_[a-z0-9_]+)\s*\(", fh.read())) - {"adn_ctx"}


def test_library_exports_every_views_header_symbol():
    import __graft_entry__ as g
    g.build()
    from adanerf_b200._lib import SYMBOLS, VIEWS_SYMBOLS
    declared = _declared("adanerf_b200_views.h")
    assert declared == set(VIEWS_SYMBOLS), declared ^ set(VIEWS_SYMBOLS)
    assert not declared & _declared("adanerf_b200.h") and not declared & set(SYMBOLS)
    lib = ctypes.CDLL(g.LIB)
    for s in declared:
        assert hasattr(lib, s), s
