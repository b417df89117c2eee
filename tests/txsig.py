"""Transactions for the sigverifyd_tx tests and tools/measure_sigverifyd_tx.py: multi-input / multi-output sv_tx records
(the shape check_tx_sig hands over for a commitment transaction), a commitment_signed-shaped workload, signing through
the device's own sighash, and the sigverifyd_tx request for a set of records."""
import ctypes

import numpy as np

from lightning_b200 import SvTx
from lightning_b200 import sigverifyd_wire as W
from tests import ecc, util

SV_TX_OUTPUTS_SERIALIZED, SV_TX_INPUTS_SERIALIZED, SV_TX_OUTPUTS_ZERO = 1, 2, 4
U32_FIELDS = ["version", "locktime", "sequence", "sighash_type", "prev_index", "flags"]
_vp, _sz = ctypes.c_void_p, ctypes.c_size_t


# the stand-alone libwally structs check_tx_sig reads (include/cln_dropin.h), for driving the drop-in through ctypes
class WallyIn(ctypes.Structure):
    _fields_ = [("txhash", ctypes.c_uint8 * 32), ("index", ctypes.c_uint32), ("sequence", ctypes.c_uint32), ("script", _vp),
                ("script_len", _sz), ("witness", _vp), ("features", ctypes.c_uint8), ("blinding_nonce", ctypes.c_uint8 * 32),
                ("entropy", ctypes.c_uint8 * 32)] + [(f, t) for f in ("issuance_amount", "inflation_keys",
                "issuance_amount_rangeproof", "inflation_keys_rangeproof") for t in (_vp, _sz)] + [("pegin_witness", _vp)]


class WallyOut(ctypes.Structure):
    _fields_ = [("satoshi", ctypes.c_uint64), ("script", _vp), ("script_len", _sz), ("features", ctypes.c_uint8)] + \
               [(f + s, t) for f in ("asset", "value", "nonce", "surjectionproof", "rangeproof") for s, t in (("", _vp), ("_len", _sz))]


class WallyTx(ctypes.Structure):
    _fields_ = [("version", ctypes.c_uint32), ("locktime", ctypes.c_uint32), ("inputs", _vp), ("num_inputs", _sz),
                ("inputs_allocation_len", _sz), ("outputs", _vp), ("num_outputs", _sz), ("outputs_allocation_len", _sz)]


class BitcoinTx(ctypes.Structure):
    _fields_ = [("wtx", ctypes.POINTER(WallyTx)), ("chainparams", _vp), ("psbt", _vp)]


def _output(rng, amount=None):
    script = b"\x00\x20" + bytes(rng.integers(0, 256, size=32, dtype=np.uint8))
    amount = int(rng.integers(330, 10**9)) if amount is None else amount
    return amount.to_bytes(8, "little") + bytes([len(script)]) + script


def make_multi_txs(rng, n, nin=(1, 4), nout=(1, 7)):
    """n transactions of nin inputs and nout outputs (ranges): serialised outputs (all of them, or for SIGHASH_SINGLE the
    one at the input's index, else SV_TX_OUTPUTS_ZERO) and, with more than one input, the serialised outpoints and
    sequences.  Returns (SvTx array, blob)."""
    txs = (SvTx * n)()
    blob = bytearray()
    for i in range(n):
        t = txs[i]
        k_in, k_out = int(rng.integers(*nin)), int(rng.integers(*nout))
        ins = [(bytes(rng.integers(0, 256, size=32, dtype=np.uint8)), int(rng.integers(0, 5)), int(rng.integers(0, 2**32)))
               for _ in range(k_in)]
        outs = [_output(rng) for _ in range(k_out)]
        me = int(rng.integers(0, k_in))
        t.version, t.locktime = 2, int(rng.integers(0, 2)) * int(rng.integers(1, 2**31))
        t.prev_txid[:] = list(ins[me][0])
        t.prev_index, t.sequence = ins[me][1], ins[me][2]
        t.sighash_type = [1, 1, 0x83, 3, 0x81][i % 5]
        t.input_amount = int(rng.integers(546, 2**45))
        ws = bytes(rng.integers(0, 256, size=int(rng.integers(71, 150)), dtype=np.uint8))
        t.script_off, t.script_len = len(blob), len(ws)
        blob += ws
        t.out_script_off = len(blob)
        if t.sighash_type & 0x1f == 3:
            if me < k_out:
                blob += outs[me]
                t.flags |= SV_TX_OUTPUTS_SERIALIZED
            else:
                t.flags |= SV_TX_OUTPUTS_ZERO
        else:
            blob += b"".join(outs)
            t.flags |= SV_TX_OUTPUTS_SERIALIZED
        t.out_script_len = len(blob) - t.out_script_off
        if k_in > 1:
            t.flags |= SV_TX_INPUTS_SERIALIZED
            t.prevouts_off = len(blob)
            blob += b"".join(txid + idx.to_bytes(4, "little") for txid, idx, _ in ins)
            t.prevouts_len = len(blob) - t.prevouts_off
            t.sequences_off = len(blob)
            blob += b"".join(seq.to_bytes(4, "little") for _, _, seq in ins)
            t.sequences_len = len(blob) - t.sequences_off
    return txs, bytes(blob)


def commitment_signed(rng, h):
    """one commitment transaction (one input, h + 2 serialised outputs, SIGHASH_ALL) and h HTLC transactions
    (util.make_htlc_txs); returns ((commitment SvTx array, blob), (HTLC SvTx array, blob))"""
    txs = (SvTx * 1)()
    t = txs[0]
    t.version, t.locktime, t.sequence, t.sighash_type = 2, 0x20000000 | int(rng.integers(0, 2**24)), 0x80000000, 1
    t.prev_txid[:] = list(rng.integers(0, 256, size=32, dtype=np.uint8))
    t.input_amount = 10**7
    ws = b"\x52\x21" + bytes(33) + b"\x21" + bytes(33) + b"\x52\xae"  # 2-of-2 funding script shape
    outs = b"".join(_output(rng) for _ in range(h + 2))
    t.script_len, t.out_script_off, t.out_script_len = len(ws), len(ws), len(outs)
    t.flags = SV_TX_OUTPUTS_SERIALIZED
    htlc = util.make_htlc_txs(rng, h)
    for i in range(h):
        htlc[0][i].sighash_type = 0x83  # anchors: SIGHASH_SINGLE|SIGHASH_ANYONECANPAY
    return (txs, ws + outs), htlc


def sign(engine, kind, sk, txs, blob):
    """signatures by sk over the device's sighash of each record (sv_verify_tx_host computes it whatever the signature);
    returns (key of `kind`, (n, 64) signatures)"""
    pub33, xy = ecc.pubkey_create(sk)
    key = pub33 if kind == 0 else xy
    n = len(txs)
    keys = np.frombuffer(key * n, np.uint8).reshape(n, len(key))
    _, sh = engine.check_tx_sigs(kind, txs, blob, keys, np.zeros((n, 64), np.uint8), want_sighash=True)
    sigs = np.frombuffer(b"".join(ecc.ecdsa_sign(sk, bytes(h)) for h in sh), np.uint8).reshape(n, 64).copy()
    return key, sigs


def spans(t, blob):
    """the four spans of record t that sigverifyd_tx carries (outpoints and sequences only for multi-input records)"""
    multi = t.flags & SV_TX_INPUTS_SERIALIZED
    cut = lambda off, ln: blob[off:off + ln]
    return (cut(t.script_off, t.script_len), cut(t.out_script_off, t.out_script_len),
            cut(t.prevouts_off, t.prevouts_len) if multi else b"", cut(t.sequences_off, t.sequences_len) if multi else b"")


def request(rid, kind, key, txs, blob, sigs, want=0):
    """the sigverifyd_tx frame for records txs (spans read from blob), one key, (n, 64) signatures"""
    n = len(txs)
    sp = [spans(t, blob) for t in txs]
    data = b"".join(b"".join(s) for s in sp)
    kw = {f: [getattr(t, f) for t in txs] for f in U32_FIELDS}
    return W.encode("sigverifyd_tx", req_id=rid, kind=kind, keylen=len(key), key=bytes(key), n=n,
                    prev_txid=b"".join(bytes(t.prev_txid) for t in txs),
                    input_amount=[t.input_amount for t in txs], output_amount=[t.output_amount for t in txs],
                    script_len=[len(s[0]) for s in sp], outputs_len=[len(s[1]) for s in sp],
                    prevouts_len=[len(s[2]) for s in sp], sequences_len=[len(s[3]) for s in sp],
                    bloblen=len(data), blob=data, sigs=np.ascontiguousarray(sigs, np.uint8).tobytes(), want_sighash=want,
                    **kw)


def expected(engine, kind, key, txs, blob, sigs):
    """(verdicts, sighashes) of the in-process engine for the same records"""
    n = len(txs)
    keys = np.frombuffer(bytes(key) * n, np.uint8).reshape(n, len(key)) if n else np.zeros((0, len(key)), np.uint8)
    return engine.check_tx_sigs(kind, txs, blob, keys, sigs, want_sighash=True)


def subset(txs, idx):
    """a fresh SvTx array holding copies of records idx (offsets still into the same blob)"""
    out = (SvTx * len(idx))()
    for j, i in enumerate(idx):
        out[j] = txs[int(i)]
    return out
