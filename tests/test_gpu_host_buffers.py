"""GPU: the context's grow-only device buffers through every host entry point that uses them.

A fresh context runs the entry points at sizes that rise, fall, then rise past the earlier maximum, interleaving entry
points whose scratch layouts differ, so that every buffer is reallocated after other entry points laid their pieces out
in it: the item staging and the launch slots' work records (sv_verify_host, samekey), the span arrays and data blob
(raw spans, SHA256d, gossip, gossip_store, transactions, BOLT11), the per-call scratch slab (gossip, transactions, mixed,
BOLT12, BOLT11, fee grind), the BOLT12 field records, the key de-duplication scratch (gossip, then BIP-340 batch) and the
distinct keys' tables.  Every output must equal the same call on a second context that first ran every entry point at
its largest size, so that none of its buffers grows during the sequence."""
import json
import os

import numpy as np
import pytest

from lightning_b200 import SvTx
from tests import bolt11, bolt12, feegrind, gossip, txsig
from tests import gossip_store as gs

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LEVELS = (1, 3, 2, 1, 4)  # rising, falling, rising past the earlier maximum
TOP = max(LEVELS)


def _synth(engine, kind, n, seed):
    """n generated signatures of `kind` (device generator), as host arrays (msg, key, sig)"""
    import torch
    keylen = {0: 33, 1: 64, 2: 32}[kind]
    t = [torch.empty((n, w), dtype=torch.uint8, device="cuda") for w in (32, keylen, 64)]
    torch.cuda.synchronize()
    engine.synth_device(kind, seed, n, *(x.data_ptr() for x in t))
    engine.sync()
    return tuple(x.cpu().numpy() for x in t)


def _inputs(engine):
    """one call per entry point and level: [(name, fn(level) -> fn(ctx) -> output)], all inputs built up front"""
    ecdsa = _synth(engine, 0, 9000 * TOP, 7500)
    schnorr = _synth(engine, 2, 4000 * TOP, 7501)
    per_kind = [_synth(engine, k, 3000 * TOP, 7510 + k) for k in range(3)]
    msgs = gossip.load_subset()
    data, off, ln, key33, sig, _, _ = gossip.items_of(msgs)
    ann = next(m for m in msgs if m[:2] == b"\x01\x00")
    flen = int.from_bytes(ann[258:260], "big")
    chain = ann[260 + flen:292 + flen]
    store = open(os.path.join(ROOT, "tests", "golden", "gossip_store_subset.bin"), "rb").read()
    recs = gs.walk(store)[0]
    fx = bolt12.load_fixture()
    fx11 = bolt11.load_fixture()
    vec = json.load(open(os.path.join(ROOT, "tests", "golden", "bolt3_htlc_txs.json")))[0]
    weight = feegrind.HTLC_SUCCESS_WEIGHT if "success" in vec["name"] else feegrind.HTLC_TIMEOUT_WEIGHT
    gtx, gblob = feegrind.htlc_tx(vec, 1, 5_000_000)
    gtx.output_amount = 5_000_000 - feegrind.fee(2070, weight)
    gkey, gsig = txsig.sign(engine, 0, (0x1234567).to_bytes(32, "big"), (SvTx * 1)(gtx), gblob)

    def verify(s):
        n = 9000 * s
        return lambda e: e.verify(0, *(a[:n] for a in ecdsa))

    def samekey(s):
        n = 9000 * s + 1
        return lambda e: e.verify_samekey(0, ecdsa[1][0], ecdsa[0][:n], ecdsa[2][:n])

    def spans(s):
        n = 1900 * s
        d = data[:int(off[n - 1] + ln[n - 1])]
        return lambda e: (e.verify_raw(0, d, off[:n], ln[:n], key33[:n], sig[:n]), e.sha256_double(d, off[:n], ln[:n]))

    def burst(s):
        # a prefix of the messages, repeated: enough repeated keys for the de-duplication path, more distinct keys each level
        part = msgs[:775 * s] * 8
        return lambda e: e.verify_gossip_burst(part, chain)

    def plain(s):
        part = msgs[:775 * s] * 4
        return lambda e: e.verify_gossip(part)

    def store_prefix(s):
        cut = store[:recs[len(recs) * s // TOP - 1][0]]
        return lambda e: e.verify_gossip_store(cut, chain)

    def tx(s):
        txs, blob = txsig.make_multi_txs(np.random.default_rng(7520 + s), 900 * s)
        return lambda e: e.check_tx_sigs(0, txs, blob, key33[:len(txs)], sig[:len(txs)], want_sighash=True)

    def mixed(s):
        c = 3000 * s
        kinds = np.repeat(np.arange(3, dtype=np.uint8), c)
        m = np.concatenate([p[0][:c] for p in per_kind])
        k = np.zeros((3 * c, 64), np.uint8)
        for kind, p in enumerate(per_kind):
            k[kind * c:(kind + 1) * c, :p[1].shape[1]] = p[1][:c]
        sg = np.concatenate([p[2][:c] for p in per_kind])
        order = np.random.default_rng(7530 + s).permutation(3 * c)
        return lambda e: e.verify_mixed(kinds[order], m[order], k[order], sg[order])

    def b12(s):
        # the fixture's streams repeated: ~0.7, 1.9, 3.1 and 4.4 MiB of field records at levels 1 to 4, so the field
        # scratch grows past its 1 MiB floor at level 3 and again at level 4
        idx = np.arange(4500 * s) % len(fx["off"])
        a = (fx["blob"], fx["off"][idx], fx["len"][idx], fx["xonly"][idx], fx["sig"][idx])
        return lambda e: (e.verify_bolt12_spans(*bolt12.NAMES[0], *a, want_sighash=True),
                          e.verify_bolt12_tagged(bolt12.NAMES, fx["names"][idx], *a, want_sighash=True))

    def b11(s):
        idx = np.arange(4000 * s) % len(fx11["off"])
        return lambda e: e.verify_bolt11_spans(fx11["blob"], fx11["off"][idx], fx11["len"][idx])

    def grind(s):
        return lambda e: e.grind_tx_fee(0, gtx, gblob, gkey, bytes(gsig[0]), weight, 253, 20000 * s)

    def batch(s):
        n = 4000 * s
        return lambda e: e.verify_schnorr_batch(*(a[:n] for a in schnorr), seed32=bytes(range(32)))

    # neighbours differ in how they carve the scratch slab; the BIP-340 batch follows the gossip de-duplication
    return [("verify", verify), ("burst", burst), ("tx", tx), ("bolt12", b12), ("grind", grind), ("store", store_prefix),
            ("mixed", mixed), ("bolt11", b11), ("spans", spans), ("plain", plain), ("grind", grind), ("batch", batch),
            ("samekey", samekey)]


def _canon(x):
    if isinstance(x, np.ndarray):
        return (x.dtype.str, x.shape, x.tobytes())
    if isinstance(x, (tuple, list)):
        return tuple(_canon(y) for y in x)
    if isinstance(x, dict):
        return tuple(sorted((k, _canon(v)) for k, v in x.items()))
    return x


def test_grow_only_buffers_rising_falling_rising(engine):
    import lightning_b200 as L
    inputs = _inputs(engine)
    calls = [(lv, name, make(lv)) for lv in LEVELS for name, make in inputs]
    fresh = L.SigVerifier(0)
    try:
        got = [_canon(fn(fresh)) for _, _, fn in calls]
    finally:
        fresh.close()
    grown = L.SigVerifier(0)
    try:
        for lv, _, fn in calls:
            if lv == TOP:
                fn(grown)
        for (lv, name, fn), g in zip(calls, got):
            assert _canon(fn(grown)) == g, (lv, name)
    finally:
        grown.close()
