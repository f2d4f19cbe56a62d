"""The C-ABI library loads and exports every symbol include/opensfm_b200.h declares
(no compute calls: there is no GPU in the CPU test environment)."""
import os
import re

from opensfm_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    txt = open(os.path.join(ROOT, "include", "opensfm_b200.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    names = set(re.findall(r"\b(osfm_[a-z0-9_]+)\s*\(", txt))
    names -= {"osfm_allreduce_fn"}
    return names


def test_library_built_in_tree():
    assert os.path.exists(_lib.LIB_PATH), "run __graft_entry__.build()"
    assert _lib.LIB_PATH.startswith(ROOT)


def test_every_declared_symbol_is_exported_and_bound():
    L = _lib.load()
    decl = _declared()
    assert len(decl) >= 35
    for name in decl:
        assert hasattr(L, name), name
    assert decl == set(_lib.SIGNATURES), decl ^ set(_lib.SIGNATURES)


def test_ba_fallback_names_match_the_header_enum():
    txt = open(os.path.join(ROOT, "include", "opensfm_b200.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    bits = {k.lower(): int(v) for k, v in re.findall(r"\bOSFM_BA_FALLBACK_([A-Z_]+)\s*=\s*(\d+)", txt)}
    assert len(bits) == 8
    assert bits == _lib.BA_FALLBACKS


def test_version_and_param_counts_without_gpu():
    L = _lib.load()
    assert L.osfm_version() >= 100
    assert [L.osfm_camera_num_params(t) for t in range(10)] == [3, 9, 3, 8, 12, 16, 1, 4, 6, 5]
    assert L.osfm_camera_num_params(11) == -1
    assert L.osfm_kernel_launch_count() >= 0


def test_product_never_imports_the_oracle():
    """A product path that routes through oracle/ voids parity: check the package sources."""
    pkg = os.path.join(ROOT, "opensfm_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f), errors="replace").read()
                assert not re.search(r"^\s*(from|import)\s+oracle", src, flags=re.M), f
