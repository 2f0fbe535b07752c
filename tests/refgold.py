"""What the unmodified reference computed in the parity tests, kept as digests (tests/golden/reference_digests.json).

The parity tests compare every result of the CUDA library with the result the reference gives for the same input.  The
reference's sources are not part of this repository, so its side of each comparison is stored: sha256 digests of the
values the test compared against, under a key naming the test and the comparison.  Pre-states that the tests hand to both
sides are built by the oracle port (oracle/ma_oracle.c), which is deterministic, so the stored digests stay valid for them.

Recording (`MAB_RECORD_REFERENCE=1`, needs oracle/_ref built from the reference's sources) runs the tests with the port in
place of the CUDA library and evaluates the reference's side of each comparison instead of looking it up; the digests are
written when the session ends (tests/golden/make_reference_digests.py).
"""
import gzip
import hashlib
import json
import os
import re

import numpy as np

RECORD = os.environ.get("MAB_RECORD_REFERENCE") == "1"
PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_digests.json")


def _feed(h, v):
    if isinstance(v, np.ndarray):
        h.update(b"A" + str(v.dtype.descr).encode() + str(v.shape).encode())
        h.update(np.ascontiguousarray(v).tobytes())
    elif isinstance(v, (bytes, bytearray)):
        h.update(b"B%d:" % len(v) + bytes(v))
    elif isinstance(v, str):
        _feed(h, v.encode())
    elif isinstance(v, (list, tuple)):
        h.update(b"L%d:" % len(v))
        for x in v:
            _feed(h, x)
    elif v is None or isinstance(v, (bool, int, float, np.integer, np.floating)):
        h.update(b"S" + repr(v if v is None or isinstance(v, bool) else (float(v) if isinstance(v, (float, np.floating)) else int(v))).encode())
    else:
        raise TypeError(f"cannot digest {type(v).__name__}")


def digest(v):
    h = hashlib.sha256()
    _feed(h, v)
    return h.hexdigest()


class Store:
    """Session-wide table key -> digest of the reference's value."""

    def __init__(self):
        self.table = json.load(open(PATH)) if os.path.exists(PATH) else {}
        self.recorded = {}

    def expect(self, key, got, want):
        """Assert that `got` (the library under test) equals the reference's value for `key`.  `want` computes the reference's
        value; it is called only when recording."""
        if RECORD:
            self.recorded[key] = digest(want())
            return
        assert key in self.table, f"no reference digest for {key} (tests/golden/make_reference_digests.py)"
        assert digest(got) == self.table[key], f"{key}: differs from the reference"

    def save(self):
        if RECORD and self.recorded:
            table = dict(self.table)
            table.update(self.recorded)
            with open(PATH, "w") as f:
                json.dump(table, f, indent=0, sort_keys=True)
                f.write("\n")


class Checker:
    """The store seen from one test: keys are the test's id and a running number (the order of its comparisons is fixed)."""

    def __init__(self, store, nodeid):
        self.store, self.nodeid, self.n = store, re.sub(r"^.*?tests/", "tests/", nodeid), 0

    def expect(self, got, want):
        self.n += 1
        self.store.expect(f"{self.nodeid}#{self.n}", got, want)

    def cli(self, how, args, got, want):
        """Outcome of a command line of the reference, compared as `how` says, keyed by its arguments (files by base name and
        content digest) so that tests which run the same command on the same input share it."""
        key = f"cli {how}: " + " ".join(_file_key(a) if os.path.isfile(a) else a for a in args)
        self.store.expect(key, got, want)


def _file_key(path):
    h = hashlib.sha256()
    op = gzip.open if path.endswith(".gz") else open       # (a gzip header carries the time it was written)
    with op(path, "rb") as f:
        for blk in iter(lambda: f.read(1 << 24), b""):
            h.update(blk)
    return f"{os.path.basename(path)}@{h.hexdigest()[:16]}"
