"""CPU-only: the BIP143 sighash of lightning_b200/csrc/sha256.cuh (host build, tests/host_emul) at every offset where the
streaming SHA-256 closes its last block, every CompactSize form, every sighash type byte and 2..64 inputs / 1..24 outputs,
against libwally's answers in tests/golden/bip143_sweep.npz (tests/bip143.py builds the cases)."""
import collections
import ctypes

import numpy as np
import pytest

from tests import bip143, util

P = util.P


@pytest.fixture(scope="module")
def sweep():
    return bip143.load()


def _desc(tx):
    return (tx.shape, hex(tx.sighash_type), len(tx.ins), len(tx.outs), tx.inp, len(tx.script), [len(s) for _, s in tx.outs][:3])


def test_sweep_reaches_the_edges(sweep):
    """the sweep has what it is for: each of the 64 final-block offsets of the prefix at least five times with a 1-byte
    CompactSize, all three CompactSize forms of the script length and of an output script, every type byte, and
    serialised outpoints / sequences ending at every offset of a block"""
    cases, _, _, fx = sweep
    htlc = [c for c in cases if c.shape == "htlc"]
    small = collections.Counter(bip143.prefix_len(len(c.script)) % 64 for c in htlc if len(c.script) < 0xfd and c.sighash_type == 1)
    assert len(small) == 64 and min(small.values()) >= 5
    lens = {len(c.script) for c in htlc}
    assert {0xfc, 0xfd, 0xffff, 0x10000, (1 << 20) + 7} <= lens
    assert {0, 0xfc, 0xfd, 0xffff, 0x10000} <= {len(c.outs[0][1]) for c in htlc}
    assert set(range(256)) <= {c.sighash_type for c in htlc}
    multi = [c for c in cases if len(c.ins) > 1]
    assert {(36 * len(c.ins)) % 64 for c in multi} >= set(range(0, 64, 4)) and {(4 * len(c.ins)) % 64 for c in multi} == set(range(0, 64, 4))
    assert fx["refused"].sum() == 3 * (256 - len(bip143.ACCEPTED) + 3)


def test_host_build_equals_libwally(emul, sweep):
    """every case: the host build's sighash equals libwally's (the model's for the python-only rows), and where libwally
    refuses the type the host build refuses it too (returns 0, zero sighash)"""
    cases, txs, blob, fx = sweep
    buf = np.frombuffer(blob, np.uint8)
    for i, tx in enumerate(cases):
        out = np.full(32, 0xee, np.uint8)
        ok = emul.emul_bip143(ctypes.byref(txs[i]), P(buf), P(out))
        if fx["refused"][i]:
            assert ok == 0 and not out.any(), ("refused type hashed", i, _desc(tx))
        else:
            assert ok == 1, ("type refused", i, _desc(tx))
            assert bytes(out) == bytes(fx["sighash"][i]), ("sighash", i, _desc(tx))


def test_model_equals_libwally(sweep):
    """tests/bip143.py equals libwally on every case libwally built, refusals included: what vouches for the model where
    the fixture's row is the model's own (python_only)"""
    cases, _, _, fx = sweep
    for i, tx in enumerate(cases):
        if not fx["python_only"][i]:
            assert (bip143.sighash(tx) or bytes(32)) == bytes(fx["sighash"][i]), (i, _desc(tx))
            assert (bip143.sighash(tx) is None) == bool(fx["refused"][i]), (i, _desc(tx))
    assert fx["python_only"].sum() < 64
