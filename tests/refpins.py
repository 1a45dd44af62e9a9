"""Bit-exact pins of the CPU oracle to the reference's own functions that need nothing outside the repository.

A pin is the SHA-256 of the bytes the reference's own code produced on seeded inputs, recorded from the libraries that
oracle/build_ref.sh compiles from the reference's source into oracle/_ref/ and stored in tests/golden/ref_pins.json with
the length of those bytes and SAMPLE_WORDS of their 32-bit words at seeded offsets. A test hashes what the oracle produces on
the same inputs and compares it with the stored digest; on a mismatch the length and the sampled words say where it
differs. Where oracle/_ref is built, the test also runs the reference itself and asserts that both give the same bytes.

After a deliberate change of a pinned test's inputs, record the digests again where oracle/_ref is built:
    REFPINS_RECORD=1 python -m pytest tests/test_oracle_vs_ref.py tests/test_oracle_vs_ref_poses.py tests/test_eval_oracle.py tests/test_frames_oracle.py tests/test_hostio.py
The decay pins need the reference's CUDA Decay, so they are recorded on the GPU:
    REFPINS_RECORD=1 python -m pytest tests/test_gpu_decay.py
"""
import atexit
import hashlib
import json
import os
import zlib

import numpy as np

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_pins.json")
RECORD = os.environ.get("REFPINS_RECORD") == "1"
SAMPLE_WORDS = 64

_golden = None
_recorded = {}


def _load():
    global _golden
    if _golden is None:
        with open(PATH) as f:
            _golden = json.load(f)["pins"]
    return _golden


def _write():
    if not _recorded:
        return
    try:
        old = _load()
    except FileNotFoundError:
        old = {}
    with open(PATH, "w") as f:
        json.dump({"what": "SHA-256, length and sampled 32-bit words (byte offset -> hex, little-endian) of the reference's own "
                           "outputs on the seeded inputs of the tests that use tests/refpins.py",
                   "pins": dict(sorted({**old, **_recorded}.items()))}, f, indent=1)
        f.write("\n")


if RECORD:
    atexit.register(_write)


def digest(b):
    return hashlib.sha256(b).hexdigest()


def _pin(b, key):
    n = len(b) // 4
    rng = np.random.default_rng(zlib.crc32(key.encode()))
    offs = sorted(int(i) * 4 for i in rng.choice(n, size=min(SAMPLE_WORDS, n), replace=False)) if n else []
    return {"sha256": digest(b), "bytes": len(b), "sample": {str(o): b[o:o + 4].hex() for o in offs}}


def _where(pin, ours):
    """The first sampled word that differs, or the length mismatch; None when every sampled word agrees."""
    if len(ours) != pin["bytes"]:
        return f"{len(ours)} bytes against the reference's {pin['bytes']}"
    for o, want in pin["sample"].items():
        got = ours[int(o):int(o) + 4].hex()
        if got != want:
            return f"at byte {o}: {got} against the reference's {want} (little-endian words)"
    return None


def check(key, ours, ref=None):
    """ours: bytes the oracle (or the project's host code) produced; ref: the same bytes from the reference's own code, or None
    where oracle/_ref is not built. Asserts ours == ref when both exist, and digest(ours) == the stored digest of the reference."""
    if ref is not None:
        assert ours == ref, f"{key}: differs from the reference's own code"
        if RECORD:
            _recorded[key] = _pin(ref, key)
            return
    pin = _load().get(key)
    assert pin is not None, f"{key}: no stored digest in {PATH}"
    if digest(ours) != pin["sha256"]:
        where = _where(pin, ours) or "outside the sampled words"
        raise AssertionError(f"{key}: differs from the stored digest of the reference's output; {where}")
