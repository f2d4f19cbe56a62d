"""Engine handles, without a GPU: every C entry point on a handle goes through the shared create / destroy helpers
or `with_handle` (null check, lock, device, error codes), and the Python handle pool hands out and takes back handles
as it should (checked with a fake create / destroy pair)."""
import ctypes
import gc
import glob
import os
import re

import pytest

from opensfm_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "opensfm_b200", "csrc")
KINDS = ("ba", "matcher", "tracks", "rotransac")
WRAPPERS = ("create_handle", "destroy_handle", "with_handle")


def _functions(src):
    """{name: (first parameter, body)} of the functions defined at file scope."""
    src = re.sub(r"//[^\n]*|/\*.*?\*/", "", src, flags=re.S)
    out = {}
    for m in re.finditer(r"^(?:static\s+)?int\s+(\w+)\s*\(([^)]*)\)\s*\{", src, flags=re.M):
        depth, i = 1, m.end()
        while depth:
            depth += {"{": 1, "}": -1}.get(src[i], 0)
            i += 1
        out[m.group(1)] = (m.group(2).split(",")[0].strip(), src[m.end():i - 1])
    return out


def _sources():
    return {os.path.basename(p): open(p).read() for p in sorted(glob.glob(os.path.join(CSRC, "*.cu")))}


def test_every_handle_entry_point_goes_through_the_shared_wrappers():
    seen = set()
    for name, src in _sources().items():
        fns = _functions(src)

        def wrapped(f, depth=0):
            body = fns[f][1]
            if any(re.search(r"\b%s\s*\(" % w, body) for w in WRAPPERS):
                return True
            # a file-local helper that takes the handle (the matcher's add_one / add_batch) counts as its body
            return depth < 2 and any(re.search(r"\b%s\s*\(\s*\w+\s*," % g, body) and wrapped(g, depth + 1)
                                     for g in fns if g != f and not g.startswith("osfm_"))

        for f, (first, _) in fns.items():
            if not f.startswith("osfm_"):
                continue
            kind = re.match(r"(?:const\s+)?osfm_(\w+)\s*\*", first)
            if kind and kind.group(1) in KINDS:
                seen.add(f)
                assert wrapped(f), "%s (%s) does not go through with_handle" % (f, name)
            for k in KINDS:
                if f == "osfm_%s_create" % k:
                    assert re.search(r"\bcreate_handle\s*\(", fns[f][1]), f
                if f == "osfm_%s_destroy" % k:
                    assert re.search(r"\bdestroy_handle\s*\(", fns[f][1]), f
        for k in KINDS:
            m = re.search(r"^struct\s+osfm_%s\b([^{;]*)\{" % k, src, flags=re.M)
            if m:
                assert re.search(r":\s*osfm::Handle<", m.group(1)), "osfm_%s is not an osfm::Handle (%s)" % (k, name)
    # only the wrappers reach into a handle: an entry point cannot touch the engine outside with_handle's lock
    for path in sorted(glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cuh"))):
        if os.path.basename(path) != "common.cuh":
            src = re.sub(r"//[^\n]*|/\*.*?\*/", "", open(path).read(), flags=re.S)
            assert not re.search(r"->\s*(impl|mu)\b", src), "%s reaches into a handle" % os.path.basename(path)
    # the parse found the entry points of all four handles
    for k in KINDS:
        assert any(f.startswith("osfm_%s_" % k) for f in seen), k
    assert len(seen) >= 60, len(seen)


class _FakeLib:
    """osfm_<kind>_create / osfm_<kind>_destroy for any kind: handles are 1, 2, 3, ... and destroys are recorded."""

    def __init__(self):
        self.created, self.destroyed = [], []

    def __getattr__(self, name):
        m = re.fullmatch(r"osfm_(\w+)_(create|destroy)", name)
        if not m:
            raise AttributeError(name)
        if m.group(2) == "create":
            def create(device, out):
                self.created.append((m.group(1), device))
                out._obj.value = len(self.created)
                return 0
            return create

        def destroy(h):
            self.destroyed.append(h.value)
            return 0
        return destroy


@pytest.fixture
def fake(monkeypatch):
    lib = _FakeLib()
    monkeypatch.setattr(_lib, "load", lambda: lib)
    monkeypatch.setattr(_lib, "_pool", {})
    return lib


def test_pool_is_last_in_first_out_per_device(fake):
    a = _lib.acquire("fake", 0)
    b = _lib.acquire("fake", 0)
    assert a is not b and fake.created == [("fake", 0), ("fake", 0)]
    _lib.release(a)
    _lib.release(b)
    assert _lib.acquire("fake", 0) is b
    assert _lib.acquire("fake", 0) is a
    c = _lib.acquire("fake", 0)
    assert c is not a and c is not b and len(fake.created) == 3


def test_pool_shares_nothing_between_devices_or_kinds(fake):
    h = _lib.acquire("fake", 0)
    _lib.release(h)
    other = _lib.acquire("fake", 1)
    assert other is not h and other.device == 1
    assert fake.created[-1] == ("fake", 1)
    assert _lib.acquire("other", 0) is not h
    assert _lib.acquire("fake", 0) is h


def test_pooled_releases_the_handle_on_an_exception(fake):
    with pytest.raises(KeyError):
        with _lib.pooled("fake", 0) as h:
            raise KeyError("boom")
    assert _lib.acquire("fake", 0) is h
    assert fake.destroyed == []


def test_a_dropped_handle_is_destroyed_once(fake):
    h = _lib.Handle("fake", 0)
    value = h.h.value
    with _lib.pooled("fake", 0) as kept:
        pass
    del h, kept
    gc.collect()
    assert fake.destroyed == [value]   # the released handle stays alive in the pool


def test_unknown_fallback_path_raises_before_a_handle_is_taken(fake):
    from opensfm_b200 import bundle, synthetic as syn

    pb = syn.scene_to_problem(syn.cube_scene(4, 50, 1.0))
    with pytest.raises(ValueError, match="no_such_path"):
        bundle.solve(pb, fallbacks=("classic_pcg", "no_such_path"))
    assert fake.created == []


def test_ptr_passes_none_through():
    assert _lib.ptr(None) is None
    import numpy as np

    a = np.zeros(3)
    assert _lib.ptr(a).value == a.ctypes.data
    assert isinstance(_lib.ptr(a), ctypes.c_void_p)
