"""Time onchaind's HTLC fee grind (onchaind/onchaind.c:389-437) four ways; prints one JSON line per case and a table.

Ranges [253, F], F in {2500, 25000, 125000} sat/kw, at weights 663 (HTLC-timeout) and 703 (HTLC-success), with the
signature's feerate at the top of the range, in the middle, or matching nowhere (signed by another key).  Per case:
  grind        sv_grind_tx_fee_host, one call (median of --reps calls after one warm-up call)
  tx_host      the same candidates (the walk up to the match) through ONE sv_verify_tx_host call, one sv_tx each:
               the engine's existing kernels only (median of --reps calls)
  dropin       onchaind's loop over the drop-in's check_tx_sig (libwally-shaped structs through ctypes), at most --cap
               calls, reported per candidate
  cln          Core Lightning's own per-candidate work on one host core, from oracle/_ref: libwally's BIP143 sighash
               (bitcoin_tx_hash_for_sig) and check_signed_hash (libsecp256k1), at most --cap candidates, per candidate
Every answer is checked against the model of the loop (tests/feegrind.py).  The card's name and power limit are read in
the same run.  Fails without a GPU.

    python tools/measure_fee_grind.py [--reps 5] [--cap 2000]
"""
import argparse
import ctypes
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from measure_bolt12 import card  # noqa: E402


def _median(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cap", type=int, default=2000)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("measure_fee_grind: no GPU")
    import lightning_b200 as L
    from lightning_b200 import SvTx, engine as E
    from tests import ecc, feegrind, txsig, util
    from tests.txsig import BitcoinTx, WallyIn, WallyOut, WallyTx

    name, power = card()
    eng = L.SigVerifier(0)
    vectors = json.load(open(os.path.join(ROOT, "tests", "golden", "bolt3_htlc_txs.json")))
    lib = ctypes.CDLL(E.LIB_PATH)
    vp, sz = ctypes.c_void_p, ctypes.c_size_t
    lib.check_tx_sig.restype = ctypes.c_bool
    lib.check_tx_sig.argtypes = [vp, sz, vp, vp, vp, vp]
    lib.cln_sigverify_set_tx_hooks.argtypes = [vp, vp]
    sizes, keep = {}, []
    hook_len = ctypes.CFUNCTYPE(sz, vp)(lambda p: sizes[p])
    hook_amt = ctypes.CFUNCTYPE(ctypes.c_uint64, vp, sz)(lambda tx, i: sizes[tx])
    lib.cln_sigverify_set_tx_hooks(ctypes.cast(hook_len, vp), ctypes.cast(hook_amt, vp))
    try:
        cln = util.load_cln()
    except RuntimeError:
        cln = None
    sk, other = bytes([0x31]) * 32, bytes([0x32]) * 32
    input_amount = 5_000_000
    rows = []
    for weight in (663, 703):
        vec = vectors[1] if weight == 663 else vectors[0]
        for top in (2500, 25000, 125000):
            for where in ("top", "middle", "none"):
                fs = top if where != "middle" else (253 + top) // 2
                t, blob = feegrind.htlc_tx(vec, 1, input_amount)
                t.output_amount = input_amount - feegrind.fee(fs, weight)
                txs = (SvTx * 1)(t)
                xy, sigs = txsig.sign(eng, 1, other if where == "none" else sk, txs, blob)
                if where == "none":
                    xy = ecc.pubkey_create(sk)[1]
                sig = bytes(sigs[0])
                want = feegrind.grind(253, top, weight, input_amount,
                                      lambda f, x: where != "none" and x == feegrind.fee(fs, weight))
                got = eng.grind_tx_fee(1, t, blob, xy, sig, weight, 253, top)
                assert got == want, (weight, top, where, got, want)
                cands = [(f, x) for f, x in feegrind.walk(253, top, weight, input_amount) if want[0] is None or f <= want[0]]
                n = len(cands)
                t_grind = _median(lambda: eng.grind_tx_fee(1, t, blob, xy, sig, weight, 253, top), a.reps)
                many = (SvTx * n)()
                for i, (_, x) in enumerate(cands):
                    many[i] = t
                    many[i].output_amount = input_amount - x
                keys = np.frombuffer(xy * n, np.uint8).reshape(n, 64)
                sg = np.frombuffer(sig * n, np.uint8).reshape(n, 64)
                v = eng.check_tx_sigs(1, many, blob, keys, sg)
                assert int(v.sum()) == (0 if where == "none" else 1) and (where == "none" or v[-1] == 1)
                t_tx = _median(lambda: eng.check_tx_sigs(1, many, blob, keys, sg), a.reps)
                # onchaind's loop over the drop-in's check_tx_sig (in process), capped
                ins = (WallyIn * 1)()
                ins[0].txhash[:] = list(bytes(t.prev_txid))
                ins[0].index, ins[0].sequence = t.prev_index, t.sequence
                outs = (WallyOut * 1)()
                os_buf = (ctypes.c_uint8 * t.out_script_len).from_buffer_copy(blob[t.out_script_off:])
                outs[0].script, outs[0].script_len = ctypes.addressof(os_buf), t.out_script_len
                w = WallyTx(t.version, t.locktime, ctypes.addressof(ins), 1, 1, ctypes.addressof(outs), 1, 1)
                tx = BitcoinTx(ctypes.pointer(w), None, None)
                ws = (ctypes.c_uint8 * t.script_len).from_buffer_copy(blob[:t.script_len])
                pub = (ctypes.c_uint8 * 64).from_buffer_copy(xy[31::-1] + xy[:31:-1])
                bsig = (ctypes.c_uint8 * 68).from_buffer_copy(sig[31::-1] + sig[:31:-1] + (1).to_bytes(4, "little"))
                keep += [ins, outs, os_buf, w, tx, ws, pub, bsig]
                sizes[ctypes.addressof(tx)], sizes[ctypes.addressof(ws)] = input_amount, t.script_len
                k = min(n, a.cap)
                lib.check_tx_sig(ctypes.addressof(tx), 0, None, ctypes.addressof(ws), ctypes.addressof(pub), ctypes.addressof(bsig))
                t0 = time.perf_counter()
                for _, x in cands[:k]:
                    outs[0].satoshi = input_amount - x
                    lib.check_tx_sig(ctypes.addressof(tx), 0, None, ctypes.addressof(ws), ctypes.addressof(pub),
                                     ctypes.addressof(bsig))
                t_dropin = (time.perf_counter() - t0) / k
                t_cln = None
                if cln is not None:
                    pub33 = ecc.pubkey_create(sk)[0]
                    t0 = time.perf_counter()
                    for _, x in cands[:k]:
                        t.output_amount = input_amount - x
                        h = util.cln_sighash(cln, t, blob)
                        cln.cln_check_signed_hash(bytes(h), sig, pub33)
                    t_cln = (time.perf_counter() - t0) / k
                row = dict(weight=weight, max_feerate=top, match=where, feerate=want[0], candidates=n,
                           grind_ms=t_grind * 1e3, grind_ns_per_candidate=t_grind / n * 1e9,
                           tx_host_ms=t_tx * 1e3, tx_host_ns_per_candidate=t_tx / n * 1e9,
                           dropin_us_per_candidate=t_dropin * 1e6,
                           cln_us_per_candidate=None if t_cln is None else t_cln * 1e6,
                           gpu=name, power_limit=power)
                rows.append(row)
                print(json.dumps(row), flush=True)
    print(f"\nGPU: {name}, power limit {power}")
    print("| weight | range | match | candidates | grind ms | tx_host ms | grind ns/cand | tx_host ns/cand | drop-in us/cand | CLN us/cand |")
    print("|---|---|---|---|---|---|---|---|---|---|")
    for r in rows:
        c = "n/a" if r["cln_us_per_candidate"] is None else f"{r['cln_us_per_candidate']:.1f}"
        print(f"| {r['weight']} | 253-{r['max_feerate']} | {r['match']} | {r['candidates']} | {r['grind_ms']:.2f} | "
              f"{r['tx_host_ms']:.2f} | {r['grind_ns_per_candidate']:.0f} | {r['tx_host_ns_per_candidate']:.0f} | "
              f"{r['dropin_us_per_candidate']:.0f} | {c} |")
    eng.close()


if __name__ == "__main__":
    main()
