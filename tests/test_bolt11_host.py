"""BOLT11 invoice signatures on the host: the fixture against the reference, and bolt11.cuh (host build) against the fixture.

tests/golden/bolt11_vectors.npz holds invoices (the BOLT #11 examples, signed invoices with and without `n`, constructed
signature and structure edge cases, flips and truncations) with Core Lightning's bolt11_decode answers
(tests/golden/make_bolt11.py).  The parse, hash and recovery code the k_b11_* kernels run is compiled for the host in
tests/host_emul (bolt11_emul.cpp) and must give CLN's status, signing hash and receiver_id for every item whose answer does
not rest on a field value the engine leaves to its caller.
"""
import collections
import ctypes

import numpy as np
import pytest

from tests import bolt11

P8 = ctypes.POINTER(ctypes.c_uint8)


@pytest.fixture(scope="module")
def fx():
    return bolt11.load_fixture()


@pytest.fixture(scope="module")
def cln11():
    return bolt11.oracle()


def _emul_run(emul, invs):
    emul.emul_bolt11.restype = ctypes.c_int
    emul.emul_bolt11.argtypes = [ctypes.c_char_p, ctypes.c_uint32, P8, P8, ctypes.POINTER(ctypes.c_int)]
    n = len(invs)
    st = np.zeros(n, np.int32)
    h = np.zeros((n, 32), np.uint8)
    node = np.zeros((n, 33), np.uint8)
    have_n = np.zeros(n, np.int32)
    for i, s in enumerate(invs):
        hn = ctypes.c_int()
        st[i] = emul.emul_bolt11(s, len(s), h[i].ctypes.data_as(P8), node[i].ctypes.data_as(P8), ctypes.byref(hn))
        have_n[i] = hn.value
    return st, h, node, have_n


def test_fixture_matches_reference(fx, cln11):
    """every item's answers are still what CLN's bolt11_decode and bolt11_decode_nosig give (replayed from the recording
    where the reference is not built)"""
    for i, s in enumerate(bolt11.invoices(fx)):
        r, node, h, f, nf = bolt11.ref_check(cln11, s)
        assert (r, node, h, f, nf) == (fx["ret"][i], fx["node"][i].tobytes(), fx["hash"][i].tobytes(), fx["fail"][i],
                                       fx["nosig_fail"][i]), i


def test_fixture_coverage(fx):
    e, lab = fx["expected"], fx["label_name"]
    assert (e == 1).sum() >= 500 and (e == 0).sum() >= 300 and (e == -1).sum() >= 500
    for name in ("signed", "signed_n", "upper", "recid23", "long", "n_wrong_len", "n_dup"):
        assert (lab == name).sum() > 0 and np.all(e[lab == name] == 1), name
    for name in ("recid_high", "r_s_range", "off_curve", "recid2_overflow"):
        assert (lab == name).sum() > 0 and np.all(e[lab == name] == 0), name
    for name in ("bech32m", "n_bad_key", "n_trailing"):
        assert (lab == name).sum() > 0 and np.all(e[lab == name] == -1), name
    # high-S: recovery accepts it, verification against `n` refuses it
    hs = lab == "high_s"
    assert (e[hs] == 1).sum() > 0 and (e[hs] == 0).sum() > 0
    assert max(fx["len"][lab == "long"]) > 2000
    # invoices refused for a field value the engine does not check stay in the corpus, counted by message
    unchecked = collections.Counter(f for f, x in zip(fx["fail"], e) if x == bolt11.UNCHECKED)
    assert sum(unchecked.values()) > 0
    assert not any(f.startswith(bolt11.SIG_REFUSALS + bolt11.STRUCTURAL) for f in unchecked), unchecked


def test_host_build_matches_fixture(fx, emul):
    """status, signing hash and receiver_id of bolt11.cuh, host build, for every item CLN's answer decides"""
    st, h, node, _ = _emul_run(emul, bolt11.invoices(fx))
    e = fx["expected"]
    m = e != bolt11.UNCHECKED
    bad = np.nonzero(m & (st != e))[0]
    assert bad.size == 0, [(int(i), fx["label_name"][i], int(st[i]), int(e[i]), fx["fail"][i]) for i in bad[:10]]
    signed = m & (e >= 0)
    np.testing.assert_array_equal(h[signed], fx["hash"][signed])
    assert not h[e == -1].any()
    ok = e == 1
    np.testing.assert_array_equal(node[ok], fx["node"][ok])
    assert not node[m & (e != 1)].any()


def test_host_build_takes_the_n_path(fx, emul):
    """the first 53-word `n` decides the path: the wrong-length and duplicate cases keep CLN's receiver_id"""
    lab = fx["label_name"]
    idx = np.nonzero(np.isin(lab, ["signed_n", "n_dup", "n_wrong_len", "signed"]))[0]
    invs = bolt11.invoices(fx)
    _, _, _, have_n = _emul_run(emul, [invs[i] for i in idx])
    want = np.isin(lab[idx], ["signed_n", "n_dup"])
    np.testing.assert_array_equal(have_n.astype(bool), want)


def test_recovery_matches_libsecp(fx, emul, cln11):
    """the recovery alone against secp256k1_ecdsa_recover: key, refusals and Q = infinity"""
    emul.emul_bolt11_recover.restype = ctypes.c_int
    emul.emul_bolt11_recover.argtypes = [ctypes.c_char_p, ctypes.c_int, ctypes.c_char_p, P8]
    out = np.zeros(33, np.uint8)
    for i in range(len(fx["recover_ok"])):
        sig, rc, msg = fx["recover_sig"][i].tobytes(), int(fx["recover_recid"][i]), fx["recover_msg"][i].tobytes()
        ok, key = bolt11.ref_recover(cln11, sig, rc, msg)
        assert (ok, key) == (fx["recover_ok"][i], fx["recover_key"][i].tobytes()), i
        got = emul.emul_bolt11_recover(sig, rc, msg, out.ctypes.data_as(P8))
        assert (got, out.tobytes()) == (ok, key), i
    assert fx["recover_ok"].sum() > 0 and (fx["recover_ok"] == 0).sum() >= 8
