"""ORACLE (test infrastructure) -- what every runner of a compiled piece of the reference shares (oracle/ref.py,
correlation_ref.py, flow_ops_ref.py, view_tools.py, vis.py and dataset_tools.py):

* `build_artefact`: compile the runner's artefact under oracle/_ref/ from the reference tree named by DEMON_REF_SRC, or
  use the one already built where that tree is absent;
* `Store`: where the artefact is absent too, the runner answers from the RESULT DIGESTS stored in one file under
  tests/golden/ (`Recorded`: shape, dtype and `digest`), keyed by the runner's own hash of the call;
* `record`: with the artefact present, DEMON_REF_RECORD=<json path> collects the digests of every call it runs.

Each runner keeps its own key function: the stored files are keyed by them.
"""
import hashlib
import json
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_GOLDEN_DIR = os.path.join(os.path.dirname(_HERE), "tests", "golden")
REF_SRC = os.environ.get("DEMON_REF_SRC", "")   # the reference's lmbspecialops/src; unset: use the stored results


def build_artefact(artefact, ref_files, deps, make_args, force=False):
    """Make `artefact` (make -C oracle -s -B <make_args> REF_SRC=...) where DEMON_REF_SRC is set and every one of
    `ref_files` exists, if it is missing, older than one of those or of `deps` (files of this directory: make does not see
    Makefile edits), or `force`.  Without the reference files: the existing artefact, or None."""
    if not (REF_SRC and all(os.path.isfile(f) for f in ref_files)):
        return artefact if os.path.isfile(artefact) else None
    deps = list(ref_files) + [os.path.join(_HERE, f) for f in deps]
    if force or not os.path.isfile(artefact) or os.path.getmtime(artefact) < max(os.path.getmtime(d) for d in deps):
        subprocess.check_call(["make", "-C", _HERE, "-s", "-B"] + list(make_args) + ["REF_SRC=" + REF_SRC])
    return artefact


def digest(a):
    """SHA-256 of the array's C-ordered bytes, floating-point arrays with every NaN replaced by the default NaN (payloads are
    not part of the contract: an x86 NaN payload is not what the GPU makes)."""
    a = np.array(a, copy=True, order="C")
    if a.dtype.kind == "f":
        a[np.isnan(a)] = np.nan
    return hashlib.sha256(a.tobytes()).hexdigest()


def entry(a):
    """The stored form of one reference output."""
    return {"shape": list(a.shape), "dtype": a.dtype.str, "sha256": digest(a)}


class Recorded:
    """Digest of a reference output, from a stored entry."""

    def __init__(self, d):
        self.shape, self.dtype, self.sha256 = tuple(d["shape"]), np.dtype(d["dtype"]), d["sha256"]

    def matches(self, a):
        a = np.asarray(a)
        return a.shape == self.shape and a.dtype == self.dtype and digest(a) == self.sha256


class Store:
    """The stored results of one runner: the JSON file `name` under tests/golden/ (or at `name`, an absolute path), read on
    first use."""

    def __init__(self, name):
        self.path = os.path.join(_GOLDEN_DIR, name)
        self._db = None

    def entries(self):
        if self._db is None:
            self._db = json.load(open(self.path)) if os.path.isfile(self.path) else {}
        return self._db

    def lookup(self, key, what):
        db = self.entries()
        if key not in db:
            raise RuntimeError("no stored %s (record it with DEMON_REF_RECORD)" % what)
        return db[key]


def record(key, value):
    """Merge `value` under `key` into the JSON file DEMON_REF_RECORD names, if it names one."""
    path = os.environ.get("DEMON_REF_RECORD")
    if not path:
        return
    db = json.load(open(path)) if os.path.isfile(path) else {}
    db[key] = value
    with open(path, "w") as f:
        json.dump(db, f, indent=0, sort_keys=True)
