"""The BIP143 (segwit v0) signature hash in plain Python, and a deterministic sweep of transactions that reaches the edges of
the device's streaming SHA-256 (lightning_b200/csrc/sha256.cuh bip143_*).

sighash() hashes a whole transaction the way libwally's bip143_signature_hash does (tx_io.c:660-757) and refuses the sighash
types wally_tx_get_input_signature_hash refuses (tx_io.c:972-1009).  It does not look at the sv_tx record built from the
transaction, so it checks the record layout too.

sweep(seed) returns the cases as Tx objects, the sv_tx records and the blob they point into:
  * prefix offsets: the HTLC shape, witness scripts of 0..320 bytes (every offset of the final block five times), the
    CompactSize form changes and 64 KiB / 1 MiB scripts;
  * hashOutputs: output scripts of 0..130 bytes and across the CompactSize forms;
  * every sighash type byte, and types with bits above the low byte;
  * 2..64 inputs (serialised outpoints and sequences across every block boundary) and 1..24 outputs, every accepted type;
  * extreme versions, locktimes, sequences, outpoint indices and amounts.
Script bytes are slices of one seeded pool, so the cases need not be stored to be rebuilt."""
import dataclasses
import hashlib
import os

import numpy as np

from lightning_b200 import SvTx

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bip143_sweep.npz")
OUTPUTS_SERIALIZED, INPUTS_SERIALIZED, OUTPUTS_ZERO = 1, 2, 4
ACP = 0x80
ACCEPTED = (0x00, 0x01, 0x02, 0x03, 0x81, 0x82, 0x83)
SATOSHI_MAX = 21 * 10**14  # libwally refuses a larger output amount (WALLY_SATOSHI_MAX)
BIG = (0x10000, 100003, (1 << 20) + 7)
ZERO32 = bytes(32)


def libwally_accepts(sighash_type):
    """wally_tx_get_input_signature_hash's switch for a Bitcoin (not Elements) segwit-v0 input (tx_io.c:972-1009): the
    six standard types and 0 (hashed like ALL); ANYPREVOUT bits (0x40, FORKID for BTC), other low bytes and any bit above
    the low byte are WALLY_EINVAL"""
    return sighash_type in ACCEPTED


def dsha(b):
    return hashlib.sha256(hashlib.sha256(b).digest()).digest()


def le(v, n):
    return int(v).to_bytes(n, "little")


def varint(v):
    """Bitcoin CompactSize"""
    if v < 0xfd:
        return bytes([v])
    if v <= 0xffff:
        return b"\xfd" + le(v, 2)
    if v <= 0xffffffff:
        return b"\xfe" + le(v, 4)
    return b"\xff" + le(v, 8)


def ser_output(amount, script):
    return le(amount, 8) + varint(len(script)) + script


@dataclasses.dataclass
class Tx:
    """one input of one transaction to sign.  shape "htlc": one input, one output, an sv_tx with flags 0; "multi": the
    serialised-span form check_tx_sig's adapter passes (outputs always serialised, outpoints and sequences when there is
    more than one input)"""
    version: int
    locktime: int
    ins: list          # (txid32, index, sequence)
    outs: list         # (amount, script)
    inp: int           # the input signed
    script: bytes      # scriptCode (the witness script)
    amount: int        # the signed input's amount
    sighash_type: int
    shape: str = "htlc"
    none_zero: bool = False  # "multi" with SIGHASH_NONE: pass SV_TX_OUTPUTS_ZERO instead of the serialised outputs

    def digest(self):
        """SHA-256 of everything the case consists of: a drifting generator changes it"""
        h = hashlib.sha256(b"bip143 case v1")
        h.update(le(self.version, 4) + le(self.locktime, 4) + le(self.inp, 4) + le(self.amount, 8) + le(self.sighash_type, 4))
        h.update(self.shape.encode() + bytes([self.none_zero]))
        h.update(le(len(self.ins), 4) + b"".join(t + le(i, 4) + le(s, 4) for t, i, s in self.ins))
        h.update(le(len(self.outs), 4) + b"".join(le(a, 8) + le(len(s), 4) + s for a, s in self.outs))
        h.update(le(len(self.script), 4) + self.script)
        return h.digest()


def sighash(tx, check=True):
    """the BIP143 sighash of input tx.inp, or None where libwally refuses the type.  check=False hashes any type with the
    same masks the device used before it refused the types libwally refuses (ANYONECANPAY = 0x80, base = type & 0x1f,
    the whole 32-bit type committed)"""
    sht = tx.sighash_type
    if check and not libwally_accepts(sht):
        return None
    acp, base = bool(sht & ACP), sht & 0x1f
    none, single = base == 2, base == 3
    hp = ZERO32 if acp else dsha(b"".join(t + le(i, 4) for t, i, _ in tx.ins))
    hs = ZERO32 if (acp or single or none) else dsha(b"".join(le(s, 4) for _, _, s in tx.ins))
    if none or (single and tx.inp >= len(tx.outs)):
        ho = ZERO32
    elif single:
        ho = dsha(ser_output(*tx.outs[tx.inp]))
    else:
        ho = dsha(b"".join(ser_output(a, s) for a, s in tx.outs))
    txid, idx, seq = tx.ins[tx.inp]
    pre = (le(tx.version, 4) + hp + hs + txid + le(idx, 4) + varint(len(tx.script)) + tx.script + le(tx.amount, 8) +
           le(seq, 4) + ho + le(tx.locktime, 4) + le(sht & 0xffffffff, 4))
    return dsha(pre)


def htlc_record(tx):
    """(SvTx with flags 0, blob) for a one-input one-output tx: the witness script, then the output script"""
    t = SvTx()
    txid, idx, seq = tx.ins[0]
    amt, os_ = tx.outs[0]
    t.version, t.locktime, t.sequence, t.sighash_type = tx.version, tx.locktime, seq, tx.sighash_type
    t.prev_txid[:] = list(txid)
    t.prev_index = idx
    t.script_off, t.script_len = 0, len(tx.script)
    t.out_script_off, t.out_script_len = len(tx.script), len(os_)
    t.input_amount, t.output_amount = tx.amount, amt
    return t, tx.script + os_


def prefix_len(script_len):
    """bytes of the preimage up to and including nSequence"""
    return 4 + 32 + 32 + 36 + len(varint(script_len)) + script_len + 8 + 4


class _Builder:
    """lays out sv_tx records over one blob: the script pool first, then each record's serialised spans"""

    def __init__(self, rng):
        self.rng = rng
        self.pool = bytes(rng.integers(0, 256, size=BIG[-1] + 4096, dtype=np.uint8))
        self.cases, self.recs = [], []
        self.tail = bytearray()

    def script(self, n):
        """n pool bytes at a seeded offset: (bytes, offset in the pool)"""
        off = int(self.rng.integers(0, len(self.pool) - n + 1)) if n <= 4096 else int(self.rng.integers(0, 4097))
        return self.pool[off:off + n], off

    def txid(self):
        return bytes(self.rng.integers(0, 256, size=32, dtype=np.uint8))

    def span(self, data):
        off = len(self.pool) + len(self.tail)
        self.tail += data
        return off

    def add(self, tx, script_off, out_off=0):
        """record tx; script_off / out_off: where its witness script / (HTLC shape) output script already lie in the pool"""
        t = SvTx()
        txid, idx, seq = tx.ins[tx.inp]
        t.version, t.locktime, t.sequence, t.sighash_type = tx.version, tx.locktime, seq, tx.sighash_type
        t.prev_txid[:] = list(txid)
        t.prev_index = idx
        t.script_off, t.script_len = script_off, len(tx.script)
        t.input_amount = tx.amount
        if tx.shape == "htlc":
            amt, os_ = tx.outs[0]
            t.out_script_off, t.out_script_len = out_off, len(os_)
            t.output_amount = amt
        else:
            base = tx.sighash_type & 0x1f
            if base == 3 and tx.inp >= len(tx.outs) or base == 2 and tx.none_zero:
                t.flags |= OUTPUTS_ZERO
                t.out_script_off = self.span(b"")
            else:
                t.flags |= OUTPUTS_SERIALIZED
                ser = ser_output(*tx.outs[tx.inp]) if base == 3 else b"".join(ser_output(a, s) for a, s in tx.outs)
                t.out_script_off, t.out_script_len = self.span(ser), len(ser)
            if len(tx.ins) > 1:
                t.flags |= INPUTS_SERIALIZED
                pv = b"".join(x + le(i, 4) for x, i, _ in tx.ins)
                t.prevouts_off, t.prevouts_len = self.span(pv), len(pv)
                sq = b"".join(le(s, 4) for _, _, s in tx.ins)
                t.sequences_off, t.sequences_len = self.span(sq), len(sq)
        self.cases.append(tx)
        self.recs.append(t)

    def htlc(self, script_len, sht, out_len=34, version=2, locktime=0, sequence=1, prev_index=1, amount=10**7,
             out_amount=9 * 10**6):
        ws, wo = self.script(script_len)
        os_, oo = self.script(out_len)
        tx = Tx(version, locktime, [(self.txid(), prev_index, sequence)], [(out_amount, os_)], 0, ws, amount, sht)
        self.add(tx, wo, oo)

    def multi(self, nin, nout, inp, sht, out_lens, script_len=71, version=2, locktime=0, amount=10**7, out_amounts=None,
              none_zero=False):
        ws, wo = self.script(script_len)
        ins = [(self.txid(), int(self.rng.integers(0, 2**32)), int(self.rng.integers(0, 2**32))) for _ in range(nin)]
        amts = out_amounts or [int(self.rng.integers(0, 2**40)) for _ in range(nout)]
        outs = [(amts[j], self.script(out_lens[j % len(out_lens)])[0]) for j in range(nout)]
        self.add(Tx(version, locktime, ins, outs, inp, ws, amount, sht, "multi", none_zero), wo)


def sweep(seed=143):
    """(cases, SvTx array, blob): every case of the module docstring, deterministic in seed"""
    b = _Builder(np.random.default_rng(seed))
    # prefix offsets: the preimage prefix is 116 + CompactSize + script bytes long
    for n in sorted(set(range(321)) | {0xfc, 0xfd, 0xfe, 0xff, 0x100, 0xfffe, 0xffff} | set(BIG)):
        for sht in (0x01, 0x83):
            b.htlc(n, sht, out_len=(0, 22, 34)[n % 3])
    # hashOutputs of the single output
    for n in list(range(131)) + [0xfc, 0xfd, 0xffff, 0x10000]:
        for sht in (0x01, 0x83):
            b.htlc(71 + n % 64, sht, out_len=n)
    # every sighash type byte, and bits above the low byte
    for n in (71, 253, 0x10000):
        for sht in list(range(256)) + [0x100, 0x80000001, 0xffffffff]:
            b.htlc(n, sht)
    # many inputs: 36-byte outpoints and 4-byte sequences crossing every block boundary
    for nin in range(2, 65):
        for sht in ACCEPTED:
            for inp in sorted({0, nin // 2, nin - 1}):
                b.multi(nin, 1 + nin % 3, inp, sht, (22, 34, 0), script_len=60 + nin)
    # many outputs of 0 / 22 / 34 / 252 / 253-byte scripts; SINGLE past the last output, NONE as SV_TX_OUTPUTS_ZERO
    for nout in range(1, 25):
        for sht in ACCEPTED:
            nin = 1 + nout % 4
            b.multi(nin, nout, nout % nin, sht, (0, 22, 34, 252, 253)[nout % 5:] + (0, 22, 34, 252, 253)[:nout % 5],
                    script_len=100 + nout, none_zero=bool(nout % 2))
        b.multi(4, nout, 3, 0x03, (22,))  # SINGLE at input 3: past the last output for nout <= 3
    # field extremes, one at a time on the HTLC shape, then the amounts pairwise
    amounts = (0, 1, SATOSHI_MAX, 1 << 63, (1 << 64) - 1)
    for sht in (0x01, 0x83):
        for v in (0, 1, 2, 0xffffffff):
            b.htlc(139, sht, version=v)
        for v in (0, 0xfffffffe, 0xffffffff):
            b.htlc(139, sht, locktime=v)
            b.htlc(139, sht, sequence=v)
        for v in (0, 0xffffffff):
            b.htlc(139, sht, prev_index=v)
    for a in amounts:
        for o in amounts:
            b.htlc(142, 0x01, amount=a, out_amount=o)
    for sht in ACCEPTED:
        for a in amounts:
            b.multi(2, 2, 1, sht, (34,), version=0xffffffff, locktime=0xffffffff, amount=a, out_amounts=[a, SATOSHI_MAX])
    txs = (SvTx * len(b.recs))(*b.recs)
    return b.cases, txs, b.pool + bytes(b.tail)


def load():
    """(cases, SvTx array, blob, fixture) for the fixture's seed, after checking that every rebuilt case is the one the
    fixture answers for.  fixture: dict of tests/golden/bip143_sweep.npz's arrays plus "refused" (libwally refuses the type;
    the sighash is zeros)"""
    with np.load(FIXTURE) as z:
        fx = {k: z[k] for k in z.files}
    cases, txs, blob = sweep(int(fx["seed"]))
    assert len(cases) == len(fx["rc"]), "tests/bip143.sweep drifted from the fixture: regenerate it"
    dg = np.frombuffer(b"".join(c.digest() for c in cases), np.uint8).reshape(-1, 32)
    bad = np.nonzero((dg != fx["digest"]).any(1))[0]
    assert bad.size == 0, f"cases {bad[:5]} differ from the fixture's (tests/golden/make_bip143_sweep.py)"
    fx["refused"] = (fx["rc"] != 0) & ~fx["python_only"]
    return cases, txs, blob, fx
