"""BOLT12 signature hashing on the host: the fixture against the reference, and bolt12.cuh (host build) against the fixture.

tests/golden/bolt12_vectors.npz holds TLV streams (real BOLT12 strings, fuzz-corpus streams, constructed edge cases) with
the reference's status, Merkle root and sighash (tests/golden/make_bolt12.py).  The parse and Merkle code the k_b12_*
kernels run is compiled for the host in tests/host_emul (bolt12_emul.cpp) and must give the same answers for every item.
"""
import ctypes

import numpy as np
import pytest

from tests import bolt12
from tests.golden.make_bolt12 import L

P8 = ctypes.POINTER(ctypes.c_uint8)


@pytest.fixture(scope="module")
def fx():
    return bolt12.load_fixture()


@pytest.fixture(scope="module")
def cln12():
    return bolt12.oracle()


def test_fixture_matches_reference(fx, cln12):
    """every item's status, root and sighash are still what CLN's fromwire_tlv / merkle_tlv / sighash_from_merkle /
    check_schnorr_sig give (replayed from the recording where the reference is not built)"""
    for i, st in enumerate(bolt12.streams(fx)):
        r, m, h = bolt12.ref_check(cln12, st, bolt12.NAMES[fx["names"][i]], fx["xonly"][i], fx["sig"][i])
        assert (r, m, h) == (fx["status"][i], fx["merkle"][i].tobytes(), fx["sighash"][i].tobytes()), i


def test_fixture_coverage(fx):
    s, lab = fx["status"], fx["label"]
    assert (s == 1).sum() >= 300 and (s == 0).sum() > 0 and (s == -1).sum() > 0
    assert np.all(s[lab == L["signed"]] == 1)
    for name in ("flip_signed_field", "wrong_key", "flip_sig", "other_name"):
        assert (lab == L[name]).sum() > 0 and np.all(s[lab == L[name]] == 0), name
    # a changed byte inside a signature-range field leaves the tree, hence the verdict, unchanged
    assert (lab == L["flip_signature_field"]).sum() > 0 and np.all(s[lab == L["flip_signature_field"]] == 1)
    assert np.all(s[lab == L["unsigned"]] == -1)
    streams = bolt12.streams(fx)
    # the constructed cases the fixture must keep: empty stream, > 5,000 fields, a value over 64 KiB, all-zero root
    assert any(len(st) == 0 for st in streams)
    assert max(len(st) for st in streams) > 65536
    assert any(st[:3] == b"\x00\x00\x01" and len(st) > 20000 for st in streams)
    zero_root = [i for i in range(len(s)) if s[i] >= 0 and not fx["merkle"][i].any()]
    assert zero_root and any(s[i] == 1 for i in zero_root)


def _emul_run(emul, fx):
    emul.emul_bolt12.restype = ctypes.c_longlong
    emul.emul_bolt12.argtypes = [ctypes.c_char_p, ctypes.c_uint32, ctypes.c_char_p, ctypes.c_uint32, P8, P8]
    n = len(fx["status"])
    st = np.zeros(n, np.int64)
    root = np.zeros((n, 32), np.uint8)
    sh = np.zeros((n, 32), np.uint8)
    for i, s in enumerate(bolt12.streams(fx)):
        mn, fn = bolt12.NAMES[fx["names"][i]]
        tag = b"lightning" + mn + fn
        st[i] = emul.emul_bolt12(s, len(s), tag, len(tag), root[i].ctypes.data_as(P8), sh[i].ctypes.data_as(P8))
    return st, root, sh


def test_host_build_matches_fixture(fx, emul):
    """parse outcome, Merkle root and sighash of bolt12.cuh, host build, for every fixture item"""
    st, root, sh = _emul_run(emul, fx)
    assert not np.any(st == -2), "the counting walk and the record walk disagree"
    np.testing.assert_array_equal(st < 0, fx["status"] < 0)
    np.testing.assert_array_equal(root, fx["merkle"])
    np.testing.assert_array_equal(sh, fx["sighash"])


def test_host_build_parse_rules(emul):
    """the parse rules one by one (wire/tlvstream.c fromwire_tlv, common/bigsize.c bigsize_get)"""
    r = bolt12.record
    cases = {
        b"": -1, r(0, b""): 1, r(1, b"a") + r(3, b"b"): 2,
        b"\xfd\x00\xfc\x00": -1, b"\xfd\x00\xfd\x00": 1, b"\xfe\x00\x00\xff\xff\x00": -1, b"\xfe\x00\x01\x00\x00\x00": 1,
        b"\xff\x00\x00\x00\x00\xff\xff\xff\xff\x00": -1, b"\xff\x00\x00\x00\x01\x00\x00\x00\x00\x00": 1,
        b"\x01\xfd\x00\x01x": -1, b"\xfd\x01": -1, b"\x01": -1, b"\x01\x02a": -1, r(1, b"") + r(1, b""): -1,
        r(2, b"") + r(1, b""): -1, r(2**64 - 2, b"") + r(2**64 - 1, b""): 2,
    }
    root, sh = np.zeros(32, np.uint8), np.zeros(32, np.uint8)
    emul.emul_bolt12.restype = ctypes.c_longlong
    for s, want in cases.items():
        got = emul.emul_bolt12(s, ctypes.c_uint32(len(s)), b"lightninginvoicesignature", ctypes.c_uint32(25),
                               root.ctypes.data_as(P8), sh.ctypes.data_as(P8))
        assert got == want, s.hex()
