"""onchaind's HTLC fee grind on the host: the feerate walk and the candidate check of verify.cuh (grind_*, the code
k_grind_setup / k_grind run), compiled into tests/host_emul, against the model of the reference loop (tests/feegrind.py)
and against Core Lightning's own BIP143 sighash and check_signed_hash on BOLT #3 HTLC transactions."""
import ctypes
import json
import os

import numpy as np
import pytest

from tests import ecc, feegrind, util

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
VECTORS = json.load(open(os.path.join(GOLD, "bolt3_htlc_txs.json")))
U64 = (1 << 64) - 1
U32 = (1 << 32) - 1
_vp, _u64 = ctypes.c_void_p, ctypes.c_uint64


def emul_walk(emul, weight, lo, hi, input_amount):
    emul.emul_grind_walk.restype = ctypes.c_size_t
    emul.emul_grind_walk.argtypes = [_u64, _u64, _u64, _u64, ctypes.c_size_t, _vp, _vp]
    n = emul.emul_grind_walk(weight, lo, hi, input_amount, 0, None, None)
    f, x = np.zeros(max(n, 1), np.uint64), np.zeros(max(n, 1), np.uint64)
    assert emul.emul_grind_walk(weight, lo, hi, input_amount, n, f.ctypes.data, x.ctypes.data) == n
    return [(int(a), int(b)) for a, b in zip(f[:n], x[:n])]


EDGES = [
    # (weight, min_feerate, max_feerate, input_amount)
    (0, 253, 5000, 10**6), (0, 0, U32, 0), (1, 253, 5000, 10**6), (999, 253, 5000, 10**6), (1000, 253, 5000, 10**6),
    (663, 253, 5000, 10**6), (703, 253, 25000, 10**9),
    (663, 4000, 4000, 10**6), (663, 4001, 4000, 10**6),            # min == max, min > max
    (1000, 1000, 2000, 1500), (663, 253, 3000, 663 * 2262 // 1000),  # a fee exactly equal to the input
    (1000, 2000, 3000, 1500), (663, 253, 300, 100),                 # the fee at min_feerate is already above the input
    (1, U32 - 5000, U32, U64), (663, 0, U32, 10000), (U32, U32 - 3, U32, U64), (1000, U32 - 10, U32, U64),
    (1, 0, 5000, 10**6), (7, 100, 3000, 10**6), (333, 0, 700, 5),  # many feerates share one fee
]


@pytest.mark.parametrize("weight,lo,hi,amount", EDGES)
def test_walk_matches_reference_loop(emul, weight, lo, hi, amount):
    assert emul_walk(emul, weight, lo, hi, amount) == list(feegrind.walk(lo, hi, weight, amount))


def _candidates(emul, kind, t, blob, key, sig, amounts):
    emul.emul_grind_candidates.argtypes = [ctypes.c_int, _vp, _vp, _vp, _vp, _vp, ctypes.c_size_t, _vp]
    a = np.array(amounts, np.uint64)
    out = np.zeros(max(len(a), 1), np.uint8)
    b = np.frombuffer(blob, np.uint8)
    emul.emul_grind_candidates(kind, ctypes.addressof(t), b.ctypes.data, bytes(key), bytes(sig), a.ctypes.data, len(a),
                               out.ctypes.data)
    return list(out[:len(a)])


def _cln_sighash(cln, t, blob, out_amount):
    t.output_amount = out_amount
    return bytes(util.cln_sighash(cln, t, blob))


def _corrupt(sig, how):
    r, s = int.from_bytes(sig[:32], "big"), int.from_bytes(sig[32:], "big")
    if how == "flip":
        return sig[:5] + bytes([sig[5] ^ 0x10]) + sig[6:]
    if how == "high_s":
        return sig[:32] + (util.N_ORDER - s).to_bytes(32, "big")
    if how == "r_zero":
        return bytes(32) + sig[32:]
    if how == "s_ge_n":
        return sig[:32] + (s + util.N_ORDER if s + util.N_ORDER < 2**256 else util.N_ORDER).to_bytes(32, "big")
    return (r + util.N_ORDER).to_bytes(32, "big") + sig[32:] if r + util.N_ORDER < 2**256 else bytes([255]) * 32 + sig[32:]


@pytest.mark.parametrize("vec", range(len(VECTORS)))
def test_candidates_match_cln(emul, cln, vec):
    """for each candidate fee around the signed one: the host build's verdict == CLN's check_signed_hash over CLN's own
    BIP143 sighash of the transaction with that output (SIGHASH_ALL and SINGLE|ANYONECANPAY, both key kinds); corrupted
    signatures verify nowhere"""
    v = VECTORS[vec]
    weight = feegrind.HTLC_SUCCESS_WEIGHT if "success" in v["name"] else feegrind.HTLC_TIMEOUT_WEIGHT
    rng = np.random.default_rng(900 + vec)
    input_amount = 5_000_000
    for sht in (1, 0x83):
        t, blob = feegrind.htlc_tx(v, sht, input_amount)
        sk = (int(rng.integers(1, 2**62)) * 7919 + vec).to_bytes(32, "big")
        pub33, xy = ecc.pubkey_create(sk)
        fs = int(rng.integers(300, 20000))
        signed_fee = feegrind.fee(fs, weight)
        sig = ecc.ecdsa_sign(sk, _cln_sighash(cln, t, blob, input_amount - signed_fee))
        cands = list(feegrind.walk(fs - 40, fs + 40, weight, input_amount))
        amounts = [input_amount - x for _, x in cands]
        hashes = [_cln_sighash(cln, t, blob, a) for a in amounts]
        want = [int(cln.cln_check_signed_hash(h, sig, pub33) == 1) for h in hashes]
        assert sum(want) == 1 and want[[x for _, x in cands].index(signed_fee)] == 1
        for kind, key in ((0, pub33), (1, xy)):
            assert _candidates(emul, kind, t, blob, key, sig, amounts) == want, (sht, kind)
        for how in ("flip", "high_s", "r_zero", "s_ge_n", "r_ge_n"):
            bad = _corrupt(sig, how)
            want_bad = [int(cln.cln_check_signed_hash(h, bad, pub33) == 1) for h in hashes[:8]]
            assert want_bad == [0] * 8
            assert _candidates(emul, 0, t, blob, pub33, bad, amounts[:8]) == want_bad, how


def test_refused_sighash_type_and_key(emul):
    """a sighash type with bits above the low byte (sv_verify_tx_host refuses it), an undecodable key: nothing verifies"""
    v = VECTORS[1]
    t, blob = feegrind.htlc_tx(v, 1, 10**6)
    sk = (12345).to_bytes(32, "big")
    pub33, xy = ecc.pubkey_create(sk)
    emul.emul_bip143.argtypes = [_vp, _vp, _vp]
    h = np.zeros(32, np.uint8)
    t.output_amount = 10**6 - 900
    emul.emul_bip143(ctypes.addressof(t), blob, h.ctypes.data)
    sig = ecc.ecdsa_sign(sk, bytes(h))
    assert _candidates(emul, 0, t, blob, pub33, sig, [10**6 - 900]) == [1]
    assert _candidates(emul, 1, t, blob, xy, sig, [10**6 - 900]) == [1]
    t.sighash_type = 0x101
    assert _candidates(emul, 0, t, blob, pub33, sig, [10**6 - 900]) == [0]
    t.sighash_type = 1
    assert _candidates(emul, 0, t, blob, bytes([4]) + pub33[1:], sig, [10**6 - 900]) == [0]
    assert _candidates(emul, 1, t, blob, xy[:63] + bytes([xy[63] ^ 1]), sig, [10**6 - 900]) == [0]


def test_exceptional_sums_with_chosen_messages(emul):
    """R = C + u1*G where u1*G = C (a doubling) verifies, and where u1*G = -C (R at infinity) does not, as the plain
    verification of the same (message, key, signature) decides; so do the crafted cases of tests/adversarial.py"""
    from tests import adversarial as adv
    emul.emul_grind_verify_msg.argtypes = [ctypes.c_int, _vp, _vp, _vp]
    emul.emul_verify_batch.argtypes = [ctypes.c_int, _vp, _vp, _vp, ctypes.c_size_t, _vp]
    cases = []
    for d in (1, 2, 3, adv.N - 1, 0xDEADBEEFCAFEBABE0123456789ABCDEF):
        for u2 in (1, 2, 7, adv.LAMBDA, adv.N - 5):
            c = adv.craft(d, u2 * d, u2)  # u1 = u2*d: u1*G = u2*Q = C, the comb's additions meet a doubling
            assert c is not None
            cases.append((c, 1))
            # u1 = -u2*d: u1*G = -C, R = infinity; any r < n, s = r/u2, m = u1*s
            r = adv.mul(12345 + u2, adv.G)[0] % adv.N
            s = min(r * adv.inv(u2, adv.N) % adv.N, adv.N - r * adv.inv(u2, adv.N) % adv.N)  # low S
            m = (adv.N - r * adv.inv(s, adv.N) * d % adv.N) * s % adv.N  # u2 = r/s
            b = lambda v: np.frombuffer(v.to_bytes(32, "big"), np.uint8)  # noqa: E731
            cases.append(((b(m), c[1], c[2], np.concatenate([b(r), b(s)])), 0))
    msgs, pub33, pubxy, sigs = adv.load()
    cases += [((msgs[i], pub33[i], pubxy[i], sigs[i]), None) for i in range(0, len(msgs), 8)]
    checked = {0: 0, 1: 0}
    for (m, p33, pxy, sg), want in cases:
        for kind, key in ((0, p33), (1, pxy)):
            plain = np.zeros(1, np.uint8)
            emul.emul_verify_batch(kind, np.ascontiguousarray(m).ctypes.data, np.ascontiguousarray(key).ctypes.data,
                                   np.ascontiguousarray(sg).ctypes.data, 1, plain.ctypes.data)
            got = emul.emul_grind_verify_msg(kind, bytes(key), bytes(sg), bytes(m))
            assert got == plain[0], (kind, want)
            if want is not None:
                assert got == want
                checked[want] += 1
    assert checked[0] >= 10 and checked[1] >= 10
