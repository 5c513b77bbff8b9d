#!/usr/bin/env python3
"""Recorded answers of the reference's own decoder (oracle/_ref: lib/decoder_impl.cc compiled against stand-in headers)
to the calls the tests make of it, so that the comparisons against the original project run on any machine.

Every call on a RefDecoder is keyed by the decoder's construction arguments and the chain of calls made on it before
(attribute name + SHA-256 of the arguments): the decoder is stateful, and a replayed call returns what the reference
returned at the same point of the same call sequence.  Arrays larger than LARGE bytes (chirp tables, long
instantaneous-frequency runs) are stored as their SHA-256 and come back as a Digest whose tobytes() compares equal only
to bytes with that digest; step records and every other result are stored whole (ref_pins.npz, compressed).

    python tests/golden/ref_replay.py      # re-record; needs oracle/_ref/liblora_ref.so (built by oracle/Makefile)
"""
from __future__ import annotations

import hashlib
import json
import os
import sys
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
DATA = HERE / "ref_pins.npz"
LARGE = 32768
RECORD_ENV = "LORA_REF_RECORD"
TESTS = "tests/test_ref_pins_oracle.py"


def _sha(b: bytes) -> str:
    return hashlib.sha256(b).hexdigest()


def _arg_key(a) -> str:
    if isinstance(a, np.ndarray):
        a = np.ascontiguousarray(a)
        return f"nd:{a.dtype.str}:{a.shape}:{_sha(a.tobytes())}"
    return repr(a)


def _chain(h: str, name: str, args) -> str:
    return _sha("|".join([h, name, *map(_arg_key, args)]).encode())


def _ctor_key(kw) -> str:
    return _sha(("ctor|" + repr(sorted(kw.items()))).encode())


class _Sha:
    """bytes of a stored array, known by digest: equal to bytes with the same SHA-256"""
    __hash__ = None

    def __init__(self, sha):
        self.sha = sha

    def __eq__(self, other):
        return isinstance(other, (bytes, bytearray)) and _sha(bytes(other)) == self.sha


class Digest:
    def __init__(self, sha, dtype, shape):
        self.sha, self.dtype, self.shape = sha, np.dtype(dtype), tuple(shape)

    def tobytes(self):
        return _Sha(self.sha)


class _Book:
    def __init__(self):
        self.index, self.arrays = {}, {}

    def enc(self, v):
        if isinstance(v, np.ndarray):
            v = np.ascontiguousarray(v)
            if v.dtype.fields is None and v.nbytes > LARGE:
                return {"sha": _sha(v.tobytes()), "dtype": v.dtype.str, "shape": list(v.shape)}
            name = f"a{len(self.arrays)}"
            self.arrays[name] = v
            return {"arr": name}
        if isinstance(v, (bytes, bytearray)):
            return {"bytes": bytes(v).hex()}
        if isinstance(v, tuple):
            return {"tuple": [self.enc(x) for x in v]}
        if isinstance(v, list):
            return [self.enc(x) for x in v]
        if isinstance(v, np.integer):
            return int(v)
        if isinstance(v, np.floating):
            return float(v)
        return v

    def dec(self, v):
        if isinstance(v, list):
            return [self.dec(x) for x in v]
        if isinstance(v, dict):
            if "arr" in v:
                return self.arrays[v["arr"]].copy()
            if "sha" in v:
                return Digest(v["sha"], v["dtype"], v["shape"])
            if "bytes" in v:
                return bytes.fromhex(v["bytes"])
            if "tuple" in v:
                return tuple(self.dec(x) for x in v["tuple"])
        return v

    def put(self, key, value):
        self.index[key] = self.enc(value)

    def get(self, key):
        if key not in self.index:
            raise KeyError("call not recorded from the reference (re-record: python tests/golden/ref_replay.py)")
        v = self.index[key]
        if isinstance(v, dict) and "raise" in v:
            raise ValueError(v["raise"])
        return self.dec(v)

    def save(self, path=DATA):
        np.savez_compressed(path, _index=np.frombuffer(json.dumps(self.index).encode(), np.uint8), **self.arrays)

    @classmethod
    def load(cls, path=DATA):
        b = cls()
        with np.load(path) as z:
            b.index = json.loads(z["_index"].tobytes().decode())
            b.arrays = {k: z[k] for k in z.files if k != "_index"}
        return b


def _is_method(name) -> bool:
    from oracle import ref as R
    return callable(getattr(R.RefDecoder, name, None))


class _Decoder:
    """A RefDecoder: the real one while recording, its recorded answers otherwise"""

    def __init__(self, book, real, **kw):
        self._book, self._real = book, real
        self._h = _ctor_key(kw)
        if real is not None:
            try:
                self._r = real.RefDecoder(**kw)
            except ValueError as e:
                book.index[self._h] = {"raise": str(e)}
                raise
            book.put(self._h, 0)
        else:
            book.get(self._h)

    def __getattr__(self, name):
        if name.startswith("_"):
            raise AttributeError(name)
        if _is_method(name):
            def call(*args):
                self._h = _chain(self._h, name, args)
                if self._real is None:
                    return self._book.get(self._h)
                v = getattr(self._r, name)(*args)
                self._book.put(self._h, v)
                return v
            return call
        self._h = _chain(self._h, name, ())
        if self._real is None:
            return self._book.get(self._h)
        v = getattr(self._r, name)
        self._book.put(self._h, v)
        return v


class RefModule:
    """The interface of oracle.ref that the tests use: RefDecoder and the integer-chain functions"""

    def __init__(self, book, real=None):
        self._book, self._real = book, real

    def RefDecoder(self, **kw):
        return _Decoder(self._book, self._real, **kw)

    def _fn(self, name, *args):
        key = _chain("fn", name, args)
        if self._real is None:
            return self._book.get(key)
        v = getattr(self._real, name)(*args)
        self._book.put(key, v)
        return v

    def rotl(self, *args):
        return self._fn("rotl", *args)

    def hamming_encode_soft(self, *args):
        return self._fn("hamming_encode_soft", *args)

    def hamming_decode_soft_byte(self, *args):
        return self._fn("hamming_decode_soft_byte", *args)


def ref_module():
    """The reference for the `ref` fixture: recording (LORA_REF_RECORD set), the compiled reference where
    oracle/_ref/liblora_ref.so exists, its recorded answers otherwise."""
    from oracle import ref as R
    if os.environ.get(RECORD_ENV):
        import atexit
        R.lib()
        book = _Book.load() if DATA.exists() and os.environ[RECORD_ENV] == "append" else _Book()
        atexit.register(book.save)
        return RefModule(book, R)
    if R.LIB.exists():
        R.lib()
        return R
    return RefModule(_Book.load())


def _record_cfo_windows(ref):
    """tests/test_gpu_stream.py::test_cfo_estimate_equals_reference_function asks the reference for the CFO of the window
    after the last SYNC step; the device's step trace equals the oracle's, so the oracle locates the same windows here."""
    sys.path.insert(0, str(HERE.parent))
    from conftest import make_capture
    from oracle import oracle as O
    for cfo_hz in (0.0, 800.0, -2500.0):
        x = make_capture(bytes.fromhex("0123456789abcdef"), 8, 4, True, seed=33, cfo_hz=cfo_hz)
        _, steps = O.Decoder(sf=8, cr=4, crc=True).run(x)
        k = int(np.nonzero(steps["state"] == 1)[0][-1])
        pos = int(steps["consumed"][: k + 1].sum())
        ref.RefDecoder(sf=8).experimental_determine_cfo(x[pos:pos + 2048])


def main():
    import subprocess
    root = HERE.parent.parent
    sys.path.insert(0, str(root))
    env = dict(os.environ, **{RECORD_ENV: "1"})
    rc = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", TESTS], cwd=root, env=env).returncode
    os.environ[RECORD_ENV] = "append"
    _record_cfo_windows(ref_module())          # saved at exit
    print("recording", DATA)
    return rc


if __name__ == "__main__":
    sys.exit(main())
