"""The reference's own outputs for the tests that compare with the original project, on every checkout.

`ref` stands in for oracle.ref. Where oracle/_ref (the reference's sources compiled by oracle/ref_build.py) exists, every call
runs the reference build; with NSB_RECORD_REF_GOLDEN=1 its results are also stored, call by call, under
tests/golden/ref/<test module>/<test>.npz. Where it does not exist (the reference's sources are not part of this repository),
the stored results of the same test are replayed, so every comparison still runs against what the reference computed.

A prebuilt library older than one of the entry points (ref.serves) replays that entry point's stored results the same way.

Results too large to store whole keep a fixed, seeded subset of their rows (axis 0: rays, coordinates, grid cells, image rows);
arrays of one call with the same number of rows keep the same rows. Such a result comes back as a `Sampled` array that knows its
rows, and `ref.match(ours, theirs)` takes the same rows of this repository's output, so the comparison runs on that sample.
Each stored call also keeps a digest of its array arguments: replaying it for different inputs fails as stale data, not as a
parity mismatch.
"""
from __future__ import annotations

import hashlib
import json
import os
import re
import zlib

import numpy as np

from oracle import ref as _ref
from oracle import ref_build

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref")
RECORD = os.environ.get("NSB_RECORD_REF_GOLDEN") == "1"
_HAVE_CPU = ref_build.build() is not None
_HAVE_CUDA = ref_build.build_cuda() is not None
MAX_FILE = 600_000  # bytes of one test's stored file; larger results keep a seeded row sample, halved until it fits


class Sampled(np.ndarray):
    """Rows `rows` (sorted indices) of a reference result with `n_rows` rows."""

    rows = None
    n_rows = 0


def _sampled(values, rows, n):
    a = np.asarray(values).view(Sampled)
    a.rows, a.n_rows = rows, n
    return a


def _digest(args, earlier=()):
    """Digest of the array arguments; an argument that is an earlier reference result of the same test (a chained call) counts by position only."""
    h = hashlib.sha256()
    for a in args:
        if isinstance(a, Sampled) or any(a is e for e in earlier):
            h.update(b"earlier reference result")
        elif isinstance(a, np.ndarray):
            h.update(str((a.shape, a.dtype.str)).encode())
            h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def _rows_for(n, k, salt):
    rng = np.random.default_rng(zlib.crc32(salt.encode()) + n)
    return np.sort(rng.choice(n, size=k, replace=False))


def _test_id():
    cur = os.environ.get("PYTEST_CURRENT_TEST", "")
    nodeid = cur.rsplit(" (", 1)[0]
    path, _, name = nodeid.partition("::")
    module = os.path.splitext(os.path.basename(path))[0]
    return module, re.sub(r"[^A-Za-z0-9_.=-]+", "_", name)


def _path(module, name):
    return os.path.join(GOLDEN, module, name + ".npz")


class _Store:
    """Results of one test, in call order."""

    def __init__(self):
        self.key = None
        self.calls = 0
        self.arrays = {}
        self.specs = []
        self.loaded = None
        self.live = []
        self.replayed = []

    def _switch(self):
        key = _test_id()
        if key != self.key:
            self.key, self.calls, self.arrays, self.specs, self.loaded, self.live, self.replayed = key, 0, {}, [], None, [], []
        return key

    def _plan(self, value, call, budget):
        """Rows to keep per axis-0 length for this call's arrays (empty: keep all)."""
        arrays = []

        def walk(v):
            if isinstance(v, np.ndarray) or type(v).__module__.startswith("torch"):
                arrays.append(v)
            elif isinstance(v, (tuple, list)):
                for x in v:
                    walk(x)
            elif isinstance(v, dict):
                for x in v.values():
                    walk(x)

        walk(value)
        total = sum(a.numel() * a.element_size() if hasattr(a, "numel") else a.nbytes for a in arrays)
        if total <= budget:
            return {}
        plan = {}
        for n in {a.shape[0] for a in arrays if len(a.shape) and a.shape[0] > 1}:
            group = [a for a in arrays if len(a.shape) and a.shape[0] == n]
            row_bytes = sum((a.numel() * a.element_size() if hasattr(a, "numel") else a.nbytes) / n for a in group)
            k = int(max(1, min(n, budget * (row_bytes * n / total) // row_bytes)))
            if k < n:
                plan[n] = _rows_for(n, k, f"{self.key}:{call}")
        return plan

    def _enc(self, v, tag, plan):
        if isinstance(v, np.ndarray) or type(v).__module__.startswith("torch"):
            kind = "a" if isinstance(v, np.ndarray) else "t"
            a = v if kind == "a" else v.detach().cpu().numpy()
            rows = plan.get(a.shape[0]) if a.ndim else None
            if rows is not None:
                self.arrays[tag] = a[rows]
                self.arrays[tag + "_rows"] = rows
                return {kind: tag, "n_rows": int(a.shape[0])}
            self.arrays[tag] = a
            return {kind: tag}
        if isinstance(v, tuple):
            return {"T": [self._enc(x, f"{tag}_{i}", plan) for i, x in enumerate(v)]}
        if isinstance(v, dict) and any(isinstance(x, np.ndarray) or type(x).__module__.startswith("torch") for x in v.values()):
            return {"D": {k: self._enc(x, f"{tag}_{k}", plan) for k, x in v.items()}}
        return {"j": v}

    def _dec(self, s, arrays, out=None):
        if "n_rows" in s:
            tag = s.get("a", s.get("t"))
            assert out is None, "a sampled reference result cannot fill the caller's buffer"
            return _sampled(arrays[tag].copy(), arrays[tag + "_rows"], s["n_rows"])
        if "a" in s:
            return arrays[s["a"]].copy()
        if "t" in s:
            import torch

            t = torch.from_numpy(arrays[s["t"]].copy()).cuda()
            if out is not None:
                out.copy_(t)
                return out
            return t
        if "T" in s:
            outs = out or [None] * len(s["T"])
            return tuple(self._dec(x, arrays, o) for x, o in zip(s["T"], outs))
        if "D" in s:
            return {k: self._dec(x, arrays) for k, x in s["D"].items()}
        return s["j"]

    def record(self, value, args):
        self._switch()
        self.live.append((value, _digest(args, self._outputs())))
        self.calls += 1
        path = _path(*self.key)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        budget = 1 << 40
        while True:
            self.arrays, self.specs = {}, []
            for call, (v, digest) in enumerate(self.live):
                spec = self._enc(v, f"c{call}", self._plan(v, call, budget / len(self.live)))
                spec["inputs"] = digest
                self.specs.append(spec)
            np.savez_compressed(path, __spec__=np.array(json.dumps(self.specs)), **self.arrays)
            if os.path.getsize(path) <= MAX_FILE:
                break
            raw = sum(a.nbytes for a in self.arrays.values())
            budget = raw / 2 if budget > raw else budget / 2

    def _outputs(self):
        out = []
        for v, _ in self.live:
            out += list(v) if isinstance(v, tuple) else [v]
        return out

    def replay(self, args, out=None):
        key = self._switch()
        if self.loaded is None:
            path = _path(*key)
            assert os.path.exists(path), (f"no stored reference results for {key[0]}::{key[1]} ({path}): record them where oracle/_ref exists "
                                          "with NSB_RECORD_REF_GOLDEN=1")
            with np.load(path) as z:
                self.loaded = (json.loads(str(z["__spec__"])), {k: z[k] for k in z.files if k != "__spec__"})
        specs, arrays = self.loaded
        assert self.calls < len(specs), f"{key}: more reference calls than were stored"
        spec = specs[self.calls]
        assert spec["inputs"] == _digest(args, self.replayed), (f"{key}: call {self.calls} has other inputs than the stored reference results "
                                                 "(stale data: record them again with NSB_RECORD_REF_GOLDEN=1)")
        v = self._dec(spec, arrays, out)
        self.calls += 1
        self.replayed += list(v) if isinstance(v, tuple) else [v]
        return v


_store = _Store()


def _call(have, fn, *args, **kw):
    inputs = list(args) + list(kw.values())
    if have:
        v = fn(*args, **kw)
        if RECORD:
            _store.record(v, inputs)
        return v
    return _store.replay(inputs)


def _stored(module):
    return os.path.isdir(os.path.join(GOLDEN, module))


class _RefCuda:
    """oracle.ref.RefCuda, or the replay of its results (render() fills the caller's fb / depth like the real one)."""

    def __init__(self, bitfield, ops=None):
        self.rc = _ref.RefCuda(bitfield, ops) if _HAVE_CUDA else None

    def close(self):
        if self.rc is not None:
            self.rc.close()

    def render(self, frame, renderer, fb=None, depth=None, stream: int = 0):
        if self.rc is not None:
            return _call(True, self.rc.render, frame, renderer, fb, depth, stream)
        return _store.replay([], out=(fb, depth, None) if fb is not None else None)

    def march_trace(self, frame, pixels, max_samples):
        return _call(_HAVE_CUDA, self.rc.march_trace if self.rc else None, frame, pixels, max_samples)

    def map_rays(self, coords):
        return _call(_HAVE_CUDA, self.rc.map_rays if self.rc else None, coords)

    def poisson_residuals(self, coords):
        return _call(_HAVE_CUDA, self.rc.poisson_residuals if self.rc else None, coords)


class _Ref:
    RefCuda = _RefCuda

    @staticmethod
    def usable(module: str) -> bool:
        """The CPU reference build exists, or results of `module`'s tests are stored."""
        return _HAVE_CPU or _stored(module)

    @staticmethod
    def cuda_usable(module: str) -> bool:
        return _HAVE_CUDA or _stored(module)

    @staticmethod
    def match(ours, theirs):
        """(ours, theirs) restricted to the rows `theirs` keeps when it is a stored sample; unchanged otherwise."""
        if not isinstance(theirs, Sampled):
            return ours, theirs
        assert ours.shape[0] == theirs.n_rows, (ours.shape, theirs.n_rows)
        plain = theirs.view(np.ndarray)
        if type(ours).__module__.startswith("torch"):
            import torch

            return ours[torch.as_tensor(theirs.rows, device=ours.device)], torch.as_tensor(plain, device=ours.device)
        return ours[theirs.rows], plain

    @staticmethod
    def fraction(theirs) -> float:
        """The share of rows a stored sample keeps (1 for a whole result): scales the tests' workload-size checks."""
        return len(theirs.rows) / theirs.n_rows if isinstance(theirs, Sampled) else 1.0

    def __getattr__(self, name):
        attr = getattr(_ref, name)
        if not callable(attr) or isinstance(attr, type) or name.startswith("_") or name in ("available", "lib", "cuda_lib", "f32", "u32", "serves"):
            return attr
        return lambda *a, **kw: _call(_HAVE_CPU and _ref.serves(name), attr, *a, **kw)


ref = _Ref()
