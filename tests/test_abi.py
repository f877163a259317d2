"""CPU: the C-ABI library builds/loads and exports every symbol include/diamond_b200.h declares (no compute calls)."""
import ctypes
import os
import re

from diamond_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    text = open(os.path.join(ROOT, "include", "diamond_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(dmd_[a-z0-9_]+)\s*\(", text)))


def test_library_built_and_loads():
    assert os.path.exists(_lib.LIB_PATH), "run __graft_entry__.build() first"
    assert _lib.lib().dmd_version() == 101


def test_every_declared_symbol_is_exported_and_bound():
    names = _declared()
    assert len(names) >= 15
    handle = ctypes.CDLL(_lib.LIB_PATH)
    for n in names:
        assert hasattr(handle, n), f"{n} declared in include/diamond_b200.h but not exported"
        assert n in _lib.SIGNATURES, f"{n} has no ctypes signature in diamond_b200/_lib.py"
    for n in _lib.SIGNATURES:
        assert n in names, f"{n} bound in _lib.py but not declared in the header"


def test_struct_sizes_match_header_layout():
    # natural alignment, 64-bit pointers: guards against field drift between the header and the ctypes mirror
    assert ctypes.sizeof(_lib.DenoiserConfigC) == 4 * 4 + 3 * 8 * 4 + 4 + 2 * 4
    assert ctypes.sizeof(_lib.ConvDesc) == 176 and ctypes.sizeof(_lib.PrepDesc) == 176
    assert ctypes.sizeof(_lib.SamplerConfigC) == 40
