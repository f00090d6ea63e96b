"""Record / replay of calls into the reference's own code (oracle/_ref, see ref_mcs_api.py, ref_match_api.py, ref_dbow2_api.py).

The tests that compare the oracle and the CUDA path with the reference reach it through `module("ref_mcs_api")` and friends.
Where MCS_RECORD_REF_TAPE=1 and the reference library is built (MCS_REFERENCE_DIR, `make -C oracle ref`), every call runs the
real library and its result is written to tests/golden/ref_tape_<test module>.{json,npz} when the session ends.  Everywhere
else the calls are answered from those files, in the order a test makes them, so the comparisons run without the reference.
The array and scalar arguments of each call are digested on recording and checked on replay: a test whose inputs drifted fails
instead of comparing against outputs of other inputs.

Arrays above a module's size limit are stored as a Digest (shape, dtype, BLAKE2b and CRC-32 of the bytes); compare them with
`same` (or `crc32` against a CRC).
With scalar_digests, floating-point results (and tuples holding one) are stored as a short digest that compares equal to an equal
value: the camera-model and fastAtan2 checks make thousands of such calls, and verbatim doubles would make the tape several times
larger.  A failing comparison against a digest shows no value; re-run the test with MCS_RECORD_REF_TAPE=1 next to the reference
library to see it.
"""
import atexit
import hashlib
import importlib
import json
import os
import pathlib
import zlib

import numpy as np

GOLD = pathlib.Path(__file__).resolve().parents[1] / "tests" / "golden"
RECORD = os.environ.get("MCS_RECORD_REF_TAPE") == "1"
# results of these calls are handles passed back into the library, never compared: replay hands out a placeholder
HANDLES = {"KF", "MPTable", "RefExtractor", "RefVocabulary", "lib"}


class Digest:
    def __init__(self, shape, dtype, hexdigest, crc32=None):
        self.shape, self.dtype, self.hexdigest, self.crc32 = tuple(shape), np.dtype(dtype), hexdigest, crc32

    def __len__(self):
        return self.shape[0]

    def __eq__(self, other):
        other = digest(other)
        return (self.shape, self.dtype.str, self.hexdigest) == (other.shape, other.dtype.str, other.hexdigest)

    def __repr__(self):
        return f"Digest({self.shape}, {self.dtype}, {self.hexdigest[:12]})"


def digest(a):
    if isinstance(a, Digest):
        return a
    a = np.ascontiguousarray(a)
    b = a.tobytes()
    return Digest(a.shape, a.dtype, hashlib.blake2b(b, digest_size=16).hexdigest(), zlib.crc32(b))


def crc32(a):
    """zlib.crc32 of an array's bytes, or the one stored with a replayed Digest"""
    return digest(a).crc32


def _value_hash(v):
    """numbers compared as Python compares them (1 == 1.0 == True), tuples element by element"""
    def norm(x):
        return tuple(norm(y) for y in x) if isinstance(x, (tuple, list)) else float(x)
    return hashlib.blake2b(repr(norm(v)).encode(), digest_size=3).hexdigest()


class ValueDigest:
    def __init__(self, h):
        self.h = h

    def __eq__(self, other):
        return self.h == (other.h if isinstance(other, ValueDigest) else _value_hash(other))

    def __repr__(self):
        return f"ValueDigest({self.h})"


def same(a, b):
    """exact equality of shape, dtype and bytes; either side may be a Digest of a replayed result"""
    return digest(a) == digest(b)


def _args_key(what, args, kwargs):
    h = hashlib.blake2b(what.encode(), digest_size=3)
    for v in list(args) + [kwargs[k] for k in sorted(kwargs)]:
        if isinstance(v, np.ndarray):
            h.update(digest(v).hexdigest.encode())
        elif isinstance(v, _Proxy):
            h.update(v._path.encode())
        elif v is None or isinstance(v, (bool, int, float, str, np.integer, np.floating)):
            h.update(repr(v).encode())
        elif isinstance(v, dict):
            h.update(_args_key("", (), v).encode())
        elif isinstance(v, (tuple, list)) and all(isinstance(x, (int, float, np.ndarray)) for x in v):
            h.update(_args_key("", v, {}).encode())
        h.update(b"|")
    return h.hexdigest()


class _Tape:
    """one file pair per test module: per test id, the digests of its calls (one string, 6 hex digits per call) and their results"""

    def __init__(self, name, limit, scalar_digests):
        self.name, self.limit, self.scalar_digests = name, limit, scalar_digests
        self.json_path, self.npz_path = GOLD / f"ref_tape_{name}.json", GOLD / f"ref_tape_{name}.npz"
        self.calls, self.arrays, self.counter = {}, {}, {}
        if RECORD:
            atexit.register(self.save)
        else:
            if not self.json_path.exists():
                raise FileNotFoundError(f"{self.json_path} is missing: record it with MCS_RECORD_REF_TAPE=1 next to the reference library")
            self.calls = json.loads(self.json_path.read_text())
            if self.npz_path.exists():
                with np.load(self.npz_path) as z:
                    self.arrays = {k: z[k] for k in z.files}

    def encode(self, key, v):
        items = v if isinstance(v, (tuple, list)) else [v]
        if self.scalar_digests and not isinstance(v, np.ndarray) and \
                all(isinstance(x, (bool, int, float, np.number, np.bool_)) for x in items) and \
                any(isinstance(x, (float, np.floating)) for x in items):
            return "#" + _value_hash(v)          # integers and booleans stay verbatim: as short as a digest, and readable
        if isinstance(v, np.ndarray):
            if v.nbytes > self.limit:
                d = digest(v)
                return {"d": [list(d.shape), d.dtype.str, d.hexdigest, d.crc32]}
            self.arrays[key] = v
            return {"a": key}
        if isinstance(v, (tuple, list)):
            return {"t" if isinstance(v, tuple) else "l": [self.encode(f"{key}.{i}", x) for i, x in enumerate(v)]}
        if isinstance(v, (np.integer, np.floating, np.bool_)):
            v = v.item()
        if v is None or isinstance(v, (bool, int, float, str)):
            return v
        raise TypeError(f"cannot record a {type(v)} result")

    def decode(self, e):
        if isinstance(e, str) and e.startswith("#"):
            return ValueDigest(e[1:])
        if not isinstance(e, dict):
            return e
        if "a" in e:
            return self.arrays[e["a"]]
        if "d" in e:
            return Digest(*e["d"])
        return (tuple if "t" in e else list)(self.decode(x) for x in e.get("t", e.get("l")))

    def call(self, what, ak, fn, args, kwargs):
        test = os.environ.get("PYTEST_CURRENT_TEST", "?").rsplit(" ", 1)[0].split("::", 1)[-1]
        n = self.counter.get(test, 0)
        self.counter[test] = n + 1
        if RECORD:
            r = fn(*args, **kwargs)
            t = self.calls.setdefault(test, {"calls": "", "results": []})
            t["calls"] += ak
            t["results"].append(self.encode(f"{test}#{n}", r))
            return r
        t = self.calls.get(test, {"calls": "", "results": []})
        assert n < len(t["results"]), f"no recorded reference call {n} ({what}) of {test} in {self.json_path.name}: re-record the tape"
        assert t["calls"][6 * n:6 * n + 6] == ak, f"call {n} ({what}) of {test} differs from the recorded one: re-record the tape"
        return self.decode(t["results"][n])

    def save(self):
        GOLD.mkdir(exist_ok=True)
        self.json_path.write_text(json.dumps(self.calls, separators=(",", ":"), sort_keys=True))
        if self.arrays:
            np.savez_compressed(self.npz_path, **self.arrays)


class _Proxy:
    def __init__(self, tape, real, path):
        self._tape, self._real, self._path = tape, real, path

    def __getattr__(self, name):
        real = getattr(self._real, name) if self._real is not None else None
        if real is not None and not callable(real):
            return real
        path = f"{self._path}.{name}"

        def call(*args, **kwargs):
            ak = _args_key(path, args, kwargs)
            args = tuple(a._real if isinstance(a, _Proxy) else a for a in args)
            kwargs = {k: (v._real if isinstance(v, _Proxy) else v) for k, v in kwargs.items()}
            if name in HANDLES:       # the handle's arguments take part in the digest of every call made through it
                return _Proxy(self._tape, real(*args, **kwargs) if RECORD else None, f"{path}[{ak}]")
            return self._tape.call(path, ak, real, args, kwargs)
        return call


_tapes = {}


def module(name, test_module, limit=256, scalar_digests=False):
    """the reference module `name` (e.g. "ref_mcs_api") as seen by the tests of `test_module`: live while recording, replayed
    from tests/golden/ref_tape_<test_module>.* otherwise"""
    real = None
    if RECORD:
        real = importlib.import_module(name)
        if not real.available():
            raise RuntimeError(f"MCS_RECORD_REF_TAPE=1 needs the reference library of {name} (make -C oracle ref)")
    if test_module not in _tapes:
        _tapes[test_module] = _Tape(test_module, limit, scalar_digests)
    return _Proxy(_tapes[test_module], real, name)
