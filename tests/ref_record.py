"""What the reference's own planner sources (oracle/_ref/libmplref.so, see oracle/ref_harness.cpp) returned in the tests that
compare against them, stored in tests/golden/reference_outputs.npz so that those comparisons also run where neither the
reference tree nor that library exists.

Every value is stored under a key that names the test and the call.  Small values (result records, short arrays) are stored
as they are; large ones (pop sequences, node tables, maps) as a SHA-256 digest of their canonical bytes, which still pins
them exactly.  Where the library is present the tests call it live and the live value must equal the stored one, so the
stored data cannot drift from the sources it was taken from.  `python tools/record_reference_outputs.py` re-records the
file (it needs the library)."""
import atexit
import hashlib
import os

import numpy as np

from oracle import ref

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_outputs.npz")
LIVE = ref.available()
RECORDING = os.environ.get("MPLB_RECORD_REFERENCE") == "1"
if RECORDING and not LIVE:
    raise RuntimeError("recording the reference's outputs needs oracle/_ref/libmplref.so")
_STORED = dict(np.load(PATH)) if os.path.exists(PATH) else {}
_NEW = {}


def _canon(a):
    a = np.ascontiguousarray(a)
    if a.dtype.names is None:
        if a.dtype.kind == "f":
            a = a.astype(np.float64)
        elif a.dtype.kind in "iub":
            a = a.astype(np.int64)
    return a


def digest(a):
    a = _canon(a)
    h = hashlib.sha256()
    h.update(("%s|%s|" % (a.dtype.str if a.dtype.names is None else a.dtype.descr, a.shape)).encode())
    h.update(a.tobytes())
    return np.array(h.hexdigest())


def _key(key):
    """Keys are namespaced by the running test (module file name and test id with its parameters)."""
    cur = os.environ.get("PYTEST_CURRENT_TEST", "").rsplit(" (", 1)[0]
    path, _, name = cur.partition("::")
    return "%s::%s/%s" % (os.path.basename(path), name, key)


def _store(key, v):
    if key in _NEW and not _equal(_NEW[key], v):
        raise AssertionError("two different values recorded under " + key)
    _NEW[key] = v


def _equal(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def value(key, live):
    """The reference's value under `key`: live() where the library exists (checked against the stored value), else the
    stored value.  For records and small arrays."""
    key = _key(key)
    if not LIVE:
        if key not in _STORED:
            raise KeyError("no stored output of the reference's sources under %r (%s)" % (key, PATH))
        return _STORED[key]
    v = np.array(live())
    if v.dtype.names and "device_ms" in v.dtype.names:
        v["device_ms"] = 0.0  # a timing, not an output
    if RECORDING:
        _store(key, v)
    else:
        assert key in _STORED and _equal(_STORED[key], v), ("stored output of the reference's sources differs from a live run", key)
    return v


def same(key, ours, live):
    """True when `ours` equals the reference's array under `key` exactly (compared live where the library exists, else by
    digest against the stored one)."""
    key = _key(key)
    if not LIVE:
        if key not in _STORED:
            raise KeyError("no stored output of the reference's sources under %r (%s)" % (key, PATH))
        return str(digest(ours)) == str(_STORED[key])
    theirs = np.asarray(live())
    d = digest(theirs)
    if RECORDING:
        _store(key, d)
    else:
        assert key in _STORED and str(_STORED[key]) == str(d), ("stored digest of the reference's sources differs from a live run", key)
    return np.array_equal(ours, theirs)


class Absent:
    """Stands in for a RefMap / RefPlanner where the library is absent: setters do nothing, and every value is read through
    `value` / `same`, which never call the live getter in that case."""

    def __getattr__(self, name):
        return lambda *a, **k: None


def _save():
    if not _NEW:
        return
    out = dict(_STORED)
    out.update(_NEW)
    tmp = PATH + ".tmp.npz"
    np.savez_compressed(tmp, **out)
    os.replace(tmp, PATH)


if RECORDING:
    atexit.register(_save)
