"""CPU: libytk_b200.so loads and exports every symbol include/yomitoku_b200.h declares (no compute calls)."""
import ctypes
import os
import re

from yomitoku_b200 import _lib, build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_builds_loads_and_exports_header_symbols():
    build.build(verbose=False)
    lib = _lib.lib()
    header = open(os.path.join(ROOT, "include", "yomitoku_b200.h")).read()
    header = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    names = sorted(set(re.findall(r"\b(ytk_[a-z0-9_]+)\s*\(", header)))
    assert len(names) >= 15
    for n in names:
        assert hasattr(lib, n), "missing export %s" % n
    for n in ("ytk_rtdetr_set_debug", "ytk_rtdetr_debug_tensor", "ytk_parseq_set_debug", "ytk_parseq_debug_tensor"):
        assert n in names                               # the stage read-out hooks are part of the header
    assert lib.ytk_version() >= 1
    assert lib.ytk_launch_count() == 0
    assert isinstance(lib.ytk_last_error(), bytes)


def test_struct_layouts_match_header():
    assert ctypes.sizeof(_lib.YtkCrop) == 32            # long long + 5 ints (+ padding)
    assert ctypes.sizeof(_lib.YtkParseqCfg) == 18 * 4    # 17 config ints + decode_ar
    assert ctypes.sizeof(_lib.YtkTensor) == 8 + 8 + 8 + 32
    assert ctypes.sizeof(_lib.YtkAttnSeq) == 32          # 4 ints + long long + 2 ints
    assert ctypes.sizeof(_lib.YtkDbRun) == 24            # 4 ints + double
    assert ctypes.sizeof(_lib.YtkArState) == 10 * 8      # ten device pointers
