"""The device's BIP143 sighash (k_bip143, k_grind_setup / k_grind) on the sweep of tests/bip143.py, against libwally's answers
in tests/golden/bip143_sweep.npz: sv_verify_tx_host, sv_grind_tx_fee_host and the verifier subdaemon's sigverifyd_tx."""
import hashlib

import numpy as np
import pytest

import lightning_b200 as L
from lightning_b200 import sigverifyd_wire as W
from tests import bip143, ecc, feegrind, txsig
from tests.sigverifyd_daemon import connect as _connect
from tests.sigverifyd_daemon import daemon  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu
SK = hashlib.sha256(b"tests/test_gpu_bip143_sweep key").digest()
MAX_FRAME = 32 + (1 << 20) * 161  # the longest frame the daemon reads (lightning_b200/csrc/sigverifyd_proto.h)
INPUT = 5_000_000


@pytest.fixture(scope="module")
def signed():
    """the sweep with one signature per case: over libwally's sighash where libwally hashes the type, else over the hash
    the device formed for that type before it refused it (tests/bip143.sighash with check=False)"""
    cases, txs, blob, fx = bip143.load()
    msgs = [bip143.sighash(c, check=False) if fx["refused"][i] else bytes(fx["sighash"][i]) for i, c in enumerate(cases)]
    sigs = np.frombuffer(b"".join(ecc.ecdsa_sign(SK, m) for m in msgs), np.uint8).reshape(-1, 64).copy()
    pub33, xy = ecc.pubkey_create(SK)
    return cases, txs, blob, fx, sigs, (pub33, xy)


def _keys(key, n):
    return np.frombuffer(bytes(key) * n, np.uint8).reshape(n, len(key))


@pytest.mark.parametrize("kind", [0, 1])
def test_verify_tx_sweep(engine, signed, kind):
    """one sv_verify_tx_host call over the whole sweep: the sighashes are libwally's (zeros where it refuses the type); a
    signature over libwally's sighash verifies, one over the hash a refused type used to get does not; after a changed
    amount or a changed script byte nothing verifies"""
    cases, txs, blob, fx, sigs, keys = signed
    n = len(cases)
    key = _keys(keys[kind], n)
    v, sh = engine.check_tx_sigs(kind, txs, blob, key, sigs, want_sighash=True)
    bad = np.nonzero((sh != fx["sighash"]).any(1))[0]
    assert bad.size == 0, [(int(i), hex(cases[i].sighash_type), cases[i].shape, len(cases[i].script)) for i in bad[:5]]
    want = (~fx["refused"]).astype(np.uint8)
    bad = np.nonzero(v != want)[0]
    assert bad.size == 0, [(int(i), hex(cases[i].sighash_type), int(v[i])) for i in bad[:5]]
    # the signed input's amount, one bit
    txs2 = txsig.subset(txs, range(n))
    for t in txs2:
        t.input_amount ^= 1
    assert not engine.check_tx_sigs(kind, txs2, blob, key, sigs).any()
    # one byte of each non-empty witness script (each position flipped once, whichever cases share it)
    flip = {txs[i].script_off + i % txs[i].script_len for i in range(n) if txs[i].script_len}
    blob2 = bytearray(blob)
    for p in flip:
        blob2[p] ^= 0x10
    v2 = engine.check_tx_sigs(kind, txs, bytes(blob2), key, sigs)
    has = np.array([t.script_len > 0 for t in txs])
    assert has.sum() > n - 10 and not v2[has].any()


def _grind_case(r, sht, out_len, feerate, weight):
    """an HTLC-shaped tx with an r-byte witness script (preimage prefix 117 + r bytes) spending INPUT, its output set to
    INPUT - fee(feerate, weight)"""
    rng = np.random.default_rng(7000 + r)
    rb = lambda k: bytes(rng.integers(0, 256, size=k, dtype=np.uint8))
    tx = bip143.Tx(2, int(rng.integers(0, 2)) * 600000, [(rb(32), int(rng.integers(0, 600)), r % 2)],
                   [(INPUT - feegrind.fee(feerate, weight), rb(out_len))], 0, rb(r), INPUT, sht)
    return tx, bip143.htlc_record(tx)


def test_grind_every_prefix_offset(engine):
    """sv_grind_tx_fee_host with the prefix (hashed once, then copied with a partly filled block into every candidate)
    ending at each of the 64 block offsets, output scripts of 0 / 22 / 34 / 253 bytes, types 0x01 and 0x83: signed at a
    chosen feerate over tests/bip143.py's sighash, the grind finds what tests/feegrind.py's walk finds"""
    offsets = set()
    for r in range(64):
        weight = (feegrind.HTLC_TIMEOUT_WEIGHT, feegrind.HTLC_SUCCESS_WEIGHT)[r % 2]
        feerate = 253 + 977 * r
        tx, (t, blob) = _grind_case(r, (0x01, 0x83)[r % 2], (0, 22, 34, 253)[r % 4], feerate, weight)
        offsets.add(bip143.prefix_len(r) % 64)
        sig = ecc.ecdsa_sign(SK, bip143.sighash(tx))
        key = ecc.pubkey_create(SK)[r % 2]
        fee = feegrind.fee(feerate, weight)
        want = feegrind.grind(253, 125000, weight, INPUT, lambda f, x: x == fee)
        assert want[1] == fee and engine.grind_tx_fee(r % 2, t, blob, key, sig, weight, 253, 125000) == want, r
    assert len(offsets) == 64


def test_grind_refused_type(engine):
    """a type libwally refuses (0x04), signed over the hash the device formed for it before refusing it: no fee is found,
    while the same transaction as SIGHASH_ALL, signed over its sighash, is found"""
    weight, feerate = feegrind.HTLC_TIMEOUT_WEIGHT, 3000
    for sht, want in ((0x04, (None, 0)), (0x01, (feerate, feegrind.fee(feerate, weight)))):
        tx, (t, blob) = _grind_case(5, sht, 34, feerate, weight)
        sig = ecc.ecdsa_sign(SK, bip143.sighash(tx, check=False))
        key = ecc.pubkey_create(SK)[0]
        assert engine.grind_tx_fee(0, t, blob, key, sig, weight, feerate, feerate + 100) == want, hex(sht)


def test_daemon_sweep(engine, signed, daemon):  # noqa: F811
    """the sweep through sigverifyd_tx requests of at most 512 records, both key kinds: sighashes and verdicts equal the
    in-process engine's.  Records are kept only while a request stays within the daemon's MAX_FRAME (a record too long
    for one frame on its own would be left out; none of the sweep is)"""
    cases, txs, blob, fx, sigs, keys = signed
    n = len(cases)
    c = _connect(daemon)
    rid = 0
    for kind in (0, 1):
        want_v, want_sh = txsig.expected(engine, kind, keys[kind], txs, blob, sigs)
        assert np.array_equal(want_v, (~fx["refused"]).astype(np.uint8))
        sent = 0
        for lo in range(0, n, 512):
            idx = np.arange(lo, min(lo + 512, n))
            frame = txsig.request(rid, kind, keys[kind], txsig.subset(txs, idx), blob, sigs[idx], 1)
            assert len(frame) <= MAX_FRAME, (lo, len(frame))
            c.sendall(frame)
            name, v = W.read_msg(c)
            assert name == "sigverifyd_tx_reply" and v["req_id"] == rid, (name, rid)
            assert np.array_equal(np.frombuffer(v["verdicts"], np.uint8), want_v[idx]), (kind, lo)
            assert v["sighashes"] == want_sh[idx].tobytes(), (kind, lo)
            rid += 1
            sent += idx.size
        assert sent == n
    c.close()
