"""CPU: the store every reference runner of the oracle falls back on (oracle/recorded.py): recording digests with
DEMON_REF_RECORD in the layout of the committed files under tests/golden/, reading them back, the digest's NaN rule, and
when a runner builds its artefact."""
import hashlib
import json
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import recorded
from oracle.recorded import Recorded, Store, digest, entry, record

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def test_record_merges_calls_into_one_file_a_store_reads_back(tmp_path, monkeypatch):
    path = tmp_path / "rec.json"
    monkeypatch.setenv("DEMON_REF_RECORD", str(path))
    a = np.arange(12, dtype=np.float32).reshape(3, 4)
    a[1, 2] = np.nan
    b = (np.arange(6) % 2).astype(np.uint8)
    record("kb", entry(b))
    record("ka", [entry(a), entry(a[:2])])
    text = path.read_text()
    db = json.loads(text)
    assert text == json.dumps(db, indent=0, sort_keys=True)
    assert sorted(db) == ["ka", "kb"]
    assert db["kb"] == {"shape": [6], "dtype": "|u1", "sha256": hashlib.sha256(b.tobytes()).hexdigest()}
    store = Store(str(path))
    assert Recorded(store.lookup("kb", "result")).matches(b)
    ra, ra2 = [Recorded(d) for d in store.lookup("ka", "result")]
    assert ra.matches(a) and ra2.matches(a[:2])
    assert not ra.matches(a[:2]) and not ra.matches(a.astype(np.float64)) and not ra.matches(a + 1)


def test_recording_a_committed_file_entry_by_entry_gives_its_bytes(tmp_path, monkeypatch):
    path = tmp_path / "rec.json"
    monkeypatch.setenv("DEMON_REF_RECORD", str(path))
    committed = Store("vis_digests.json").entries()
    assert committed
    for k in reversed(sorted(committed)):
        record(k, committed[k])
    assert path.read_bytes() == open(os.path.join(GOLDEN, "vis_digests.json"), "rb").read()


def test_record_without_the_variable_writes_nothing(tmp_path, monkeypatch):
    monkeypatch.delenv("DEMON_REF_RECORD", raising=False)
    monkeypatch.chdir(tmp_path)
    record("k", entry(np.zeros(3)))
    assert os.listdir(tmp_path) == []


@pytest.mark.parametrize("dtype, nan_bits", [(np.float32, (0x7fc00001, 0xffc00000, 0x7f800001)),
                                             (np.float64, (0x7ff8000000000001, 0xfff8000000000000, 0x7ff0000000000001))])
def test_digest_ignores_nan_payloads_only(dtype, nan_bits):
    u = np.uint32 if dtype == np.float32 else np.uint64
    a = np.array([1.5, np.nan, -0.0, np.inf, np.nan], dtype=dtype)
    for bits in nan_bits:
        b = a.copy()
        b.view(u)[1] = bits
        b.view(u)[4] = bits
        assert np.isnan(b[1]) and b.view(u)[1] != a.view(u)[1]
        assert digest(b) == digest(a)
    c = a.copy()
    c[2] = 0.0                                   # -0 and +0 differ in their bits, so in the digest
    assert digest(c) != digest(a)
    finite = np.array([[1.0, 2.5], [3.0, -4.0]], dtype=dtype)
    assert digest(finite) == hashlib.sha256(finite.tobytes()).hexdigest()
    assert digest(finite.T) == hashlib.sha256(np.ascontiguousarray(finite.T).tobytes()).hexdigest()


def test_digest_hashes_integer_arrays_as_their_bytes():
    m = np.array([[0, 1, 255], [7, 0, 1]], dtype=np.uint8)
    assert digest(m) == hashlib.sha256(m.tobytes()).hexdigest()


def test_a_missing_key_raises(tmp_path):
    path = tmp_path / "db.json"
    path.write_text(json.dumps({"k": {"shape": [1], "dtype": "<f4", "sha256": "0"}}))
    with pytest.raises(RuntimeError, match=r"no stored result for this op call \(record it with DEMON_REF_RECORD\)"):
        Store(str(path)).lookup("other", "result for this op call")
    absent = Store(str(tmp_path / "absent.json"))
    assert absent.entries() == {}
    with pytest.raises(RuntimeError):
        absent.lookup("k", "result")


def test_build_artefact_uses_what_exists_and_rebuilds_what_is_stale(tmp_path, monkeypatch):
    calls = []
    monkeypatch.setattr(recorded.subprocess, "check_call", lambda args: calls.append(args))
    artefact, src = tmp_path / "lib.so", tmp_path / "src.cc"
    build = lambda force=False: recorded.build_artefact(str(artefact), [str(src)], ["Makefile"], ["-f", "x.mk", "x"], force)
    # no reference tree: the artefact if it exists, else None, and never make
    monkeypatch.setattr(recorded, "REF_SRC", "")
    assert build() is None
    artefact.write_bytes(b"")
    assert build() == str(artefact) and build(force=True) == str(artefact)
    monkeypatch.setattr(recorded, "REF_SRC", str(tmp_path))
    assert build() == str(artefact)              # a reference file is missing
    assert calls == []
    # the reference tree present: make when the artefact is older than a reference or repository file, or when forced
    src.write_text("")
    os.utime(artefact, (0, 0))
    assert build() == str(artefact)
    future = max(os.path.getmtime(src), os.path.getmtime(os.path.join(os.path.dirname(recorded.__file__), "Makefile"))) + 100
    os.utime(artefact, (future, future))
    assert build() == str(artefact)
    assert build(force=True) == str(artefact)
    make = ["make", "-C", os.path.dirname(recorded.__file__), "-s", "-B", "-f", "x.mk", "x", "REF_SRC=" + str(tmp_path)]
    assert calls == [make, make]
