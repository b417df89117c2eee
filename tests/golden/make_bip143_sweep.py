"""Generate tests/golden/bip143_sweep.npz: libwally's answer for every case of tests/bip143.sweep().

Needs oracle/_ref/libcln_ref.so (oracle/Makefile, from a Core Lightning source tree).  The cases are rebuilt from the seed,
so only the answers are stored:
  * one-input one-output cases (every sighash type byte among them): cln_htlc_sighash, which returns libwally's return code
    (wally_tx_get_btc_signature_hash with WALLY_TX_FLAG_USE_WITNESS);
  * the multi-input / multi-output cases: cln_tx_new / cln_tx_add_input / cln_tx_add_output and cln_tx_sighash
    (bitcoin_tx_hash_for_sig itself), accepted types only, since bitcoin_tx_hash_for_sig asserts on the others.
A case libwally will not build (an output amount above WALLY_SATOSHI_MAX) is marked python_only and its sighash is taken from
tests/bip143.py.

Arrays (n cases): rc (int32: libwally's return code, 0 where it hashed), sighash (n, 32; zeros where libwally refuses the
type), python_only (bool), digest (n, 32: tests.bip143.Tx.digest of each case), seed.
Run:  python -m tests.golden.make_bip143_sweep
"""
import ctypes
import io
import os
import sys
import zipfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tests import bip143, util  # noqa: E402

SEED = 143
OUT = os.path.join(ROOT, "tests", "golden", "bip143_sweep.npz")


def _lib():
    cln = util.load_cln()
    vp, u32, u64, sz, p = ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint64, ctypes.c_size_t, ctypes.c_char_p
    cln.cln_htlc_sighash.argtypes = [u32, u32, p, u32, u32, p, sz, u64, u64, p, sz, u32, vp]
    cln.cln_tx_new.restype = vp
    cln.cln_tx_new.argtypes = [u32, u32]
    cln.cln_tx_add_input.argtypes = [vp, p, u32, u32]
    cln.cln_tx_add_output.argtypes = [vp, u64, p, sz]
    cln.cln_tx_free.argtypes = [vp]
    cln.cln_tx_set_input_amount.argtypes = [u64]
    cln.cln_tal_bytes.restype = vp
    cln.cln_tal_bytes.argtypes = [p, sz]
    cln.cln_tal_free.argtypes = [vp]
    cln.cln_tx_sighash.argtypes = [vp, ctypes.c_uint, vp, u32, vp]
    return cln


def libwally(cln, tx):
    """(rc, sighash, python_only) of one case"""
    out = ctypes.create_string_buffer(32)
    nul = lambda b: b or None  # libwally takes NULL, not an empty buffer, for an empty span
    if tx.shape == "htlc":
        txid, idx, seq = tx.ins[0]
        amt, os_ = tx.outs[0]
        rc = cln.cln_htlc_sighash(tx.version, tx.locktime, txid, idx, seq, nul(tx.script), len(tx.script), tx.amount, amt,
                                  nul(os_), len(os_), tx.sighash_type, out)
        if rc and bip143.libwally_accepts(tx.sighash_type):
            return rc, bip143.sighash(tx), True  # refused for a reason other than the type: the model answers
        return rc, out.raw if rc == 0 else bytes(32), False
    assert bip143.libwally_accepts(tx.sighash_type), "bitcoin_tx_hash_for_sig asserts on a refused type"
    h = cln.cln_tx_new(tx.version, tx.locktime)
    try:
        for txid, idx, seq in tx.ins:
            assert cln.cln_tx_add_input(h, txid, idx, seq) == 0
        for amt, sc in tx.outs:
            rc = cln.cln_tx_add_output(h, amt, nul(sc), len(sc))
            if rc:
                return rc, bip143.sighash(tx), True
        ws = cln.cln_tal_bytes(tx.script, len(tx.script))
        cln.cln_tx_set_input_amount(tx.amount)
        cln.cln_tx_sighash(h, tx.inp, ws, tx.sighash_type, out)
        cln.cln_tal_free(ws)
    finally:
        cln.cln_tx_free(h)
    return 0, out.raw, False


def save(path, arrays):
    """np.savez_compressed with fixed member timestamps, so that the file is the same on every run"""
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as z:
        for k in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(arrays[k]), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            info.external_attr = 0o644 << 16
            z.writestr(info, buf.getvalue())


def main():
    cln = _lib()
    cases, _, _ = bip143.sweep(SEED)
    n = len(cases)
    rc = np.zeros(n, np.int32)
    sh = np.zeros((n, 32), np.uint8)
    py = np.zeros(n, bool)
    dg = np.zeros((n, 32), np.uint8)
    for i, tx in enumerate(cases):
        r, h, p = libwally(cln, tx)
        rc[i], py[i] = r, p
        sh[i] = np.frombuffer(h, np.uint8)
        dg[i] = np.frombuffer(tx.digest(), np.uint8)
        if not p:  # the model must agree wherever libwally answered
            assert (bip143.sighash(tx) or bytes(32)) == h, (i, hex(tx.sighash_type), tx.shape, len(tx.script))
    save(OUT, dict(rc=rc, sighash=sh, python_only=py, digest=dg, seed=np.array(SEED, np.int64)))
    print(f"{n} cases: {(rc == 0).sum()} hashed by libwally, {((rc != 0) & ~py).sum()} types refused, {py.sum()} python-only; "
          f"{os.path.getsize(OUT)} bytes")


if __name__ == "__main__":
    main()
