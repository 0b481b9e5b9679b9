"""The C-ABI shared library loads and exports exactly what include/e4s_b200.h declares (no GPU needed)."""
import ctypes
import os
import re

from conftest import ROOT


def _header_functions():
    text = open(os.path.join(ROOT, "include", "e4s_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(e4s_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    import __graft_entry__ as entry
    entry.build()
    from e4s_b200 import _lib
    lib = ctypes.CDLL(_lib.LIB_PATH)
    declared = _header_functions()
    assert len(declared) >= 15
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/e4s_b200.h but not exported"
    assert sorted(_lib.exported_symbols()) == declared, "ctypes table and header disagree"


def test_version_and_arch_strings():
    from e4s_b200 import _lib
    lib = _lib.load()
    assert lib.e4s_version() >= 100
    assert lib.e4s_build_arch() == b"sm_90a"


def test_sass_is_sm90a_only():
    import subprocess
    from e4s_b200 import _lib
    out = subprocess.run(["cuobjdump", "-lelf", _lib.LIB_PATH], capture_output=True, text=True).stdout
    archs = set(re.findall(r"sm_(\d+a?)", out))
    assert archs == {"90a"}, archs


def test_gradient_kernel_work_list_plan(monkeypatch):
    """csrc/modconv_tc.cu: N-tile width and region-pass / parity split chosen per shape (host-only entry point; the SM count
    falls back to 132, an H100 SXM, without a device).  The shapes are the layers of the 1024x1024 generator."""
    from e4s_b200 import _lib
    lib = _lib.load()
    for var in ("E4S_B200_NTILE", "E4S_B200_DGRAD_SPLIT"):
        monkeypatch.delenv(var, raising=False)

    def plan(batch, res, cin, ncls, up):
        nt, g, h = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
        assert lib.e4s_modconv3x3_bwd_tc_plan(batch, res, res, cin, ncls, int(up), ctypes.byref(nt), ctypes.byref(g), ctypes.byref(h)) == 0
        return nt.value, g.value, h.value

    # one face (the inversion loop): the low-resolution 512-channel layers take the narrow channel tile and are cut into
    # region passes (~4 work items per SM)
    assert plan(1, 4, 512, 12, True) == (32, 12, 1)         # c0: 16 (tile, channel tile) pairs -> 192 work items
    assert plan(1, 4, 512, 12, False) == (32, 12, 1)        # conv1
    assert plan(1, 32, 512, 12, False) == (32, 5, 1)        # c5: 96 pairs -> 480 items
    assert plan(1, 64, 512, 12, True) == (64, 3, 1)         # c8: 256 pairs -> 768 items
    # enough pairs: untouched
    assert plan(1, 256, 128, 1, True) == (64, 1, 1)         # c12 (no label map above 256x256)
    assert plan(1, 1024, 32, 1, False) == (32, 1, 1)        # c15
    assert plan(16, 64, 512, 12, False) == (64, 1, 1)       # a 16-face batch at 64x64: 2048 pairs
    # a 16-face batch at 4x4 still splits (128 pairs)
    assert plan(16, 4, 512, 12, False) == (64, 5, 1)
    assert lib.e4s_modconv3x3_bwd_tc_plan(1, 4, 4, 48, 12, 0, None, None, None) == -1

    # E4S_B200_NTILE forces 32 or 64; another width leaves the automatic choice
    shapes = [(1, 4, 512, 12, True), (1, 64, 512, 12, True), (16, 4, 512, 12, False)]
    auto = [plan(*a) for a in shapes]
    for ntile in ("128", "256"):
        monkeypatch.setenv("E4S_B200_NTILE", ntile)
        assert [plan(*a) for a in shapes] == auto, ntile
    monkeypatch.setenv("E4S_B200_NTILE", "32")
    assert plan(1, 64, 512, 12, True) == (32, 1, 1)          # c8: 64 by default
    assert plan(16, 4, 512, 12, False) == (32, 3, 1)
