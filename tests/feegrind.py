"""onchaind's HTLC fee grind (onchaind/onchaind.c:389-437) as a model for the tests, and the HTLC transactions it runs on.

grind_htlc_tx_fee walks every feerate from min_possible_feerate to max_possible_feerate: fee = feerate * weight / 1000
(amount_tx_fee, common/amount.c:698-707), a fee equal to the previous one is skipped, the first fee above the input amount
ends the walk, and the first fee whose transaction (output = input - fee) verifies is the answer."""
from lightning_b200 import SvTx

HTLC_TIMEOUT_WEIGHT, HTLC_SUCCESS_WEIGHT = 663, 703  # BOLT #3 without anchors (706 / 666 with option_anchor_outputs)


def fee(feerate, weight):
    return feerate * weight // 1000


def walk(min_feerate, max_feerate, weight, input_amount):
    """the (feerate, fee) pairs the reference loop checks, in its order"""
    prev = None
    for f in range(min_feerate, max_feerate + 1):
        x = fee(f, weight)
        if x == prev:
            if weight == 0:  # every later feerate repeats fee 0: the loop only skips from here on
                return
            continue
        prev = x
        if x > input_amount:
            return
        yield f, x


def grind(min_feerate, max_feerate, weight, input_amount, verifies):
    """the reference loop with verifies(feerate, fee) -> bool standing for check_tx_sig: (feerate, fee) or (None, 0)"""
    for f, x in walk(min_feerate, max_feerate, weight, input_amount):
        if verifies(f, x):
            return f, x
    return None, 0


def htlc_tx(vec, sighash_type=1, input_amount=None):
    """an SvTx (flags 0) and its script blob from one tests/golden/bolt3_htlc_txs.json entry"""
    ws, os_ = bytes.fromhex(vec["wscript"]), bytes.fromhex(vec["out_script"])
    t = SvTx()
    t.version, t.locktime, t.sequence, t.sighash_type = vec["version"], vec["locktime"], vec["sequence"], sighash_type
    t.prev_txid[:] = list(bytes.fromhex(vec["prev_txid"]))
    t.prev_index = vec["prev_index"]
    t.script_off, t.script_len = 0, len(ws)
    t.out_script_off, t.out_script_len = len(ws), len(os_)
    t.input_amount = vec["input_amount"] if input_amount is None else input_amount
    return t, ws + os_
