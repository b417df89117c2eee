"""Python model of sv_prune_gossip_store_host and sv_prune_gossip_store_funding_host: which records of a gossip_store to
mark deleted so that gossipd's strict load (common/gossmap.c with expected_len, :1428-1438) accepts the store and keeps
every record that verifies.  Built on the audit's model (tests/gossip_store.py) and, with a funding table, the funding
check's (tests/gossip_store_funding.py); the rules are those of include/cln_sigverify.h."""
from tests import gossip_store_funding as gf
from tests.gossip_store import (
    BAD_CRC, CHANNEL_AMOUNT, DELETED, HDR, NO_AMOUNT, NOT_REACHED, STORE_RECORD, STORE_TYPES, TRUNCATED, UNKNOWN, crc_ok,
    holders, signer, walk)

# reasons (include/cln_sigverify.h SV_GP_*; 0 = kept), and the summary's name of each from GP_BAD_CRC on
(GP_KEPT, GP_BAD_CRC, GP_TRUNCATED, GP_MESSAGE, GP_REDUNDANT, GP_NO_CHANNEL, GP_SIGNATURE, GP_AMOUNT, GP_UNKNOWN,
 GP_FUNDING) = range(10)
REASONS = ("bad_crc", "truncated", "message", "redundant", "no_channel", "signature", "amount", "unknown")


def prune(store, sigcheck=None, table=None):
    """-> (pruned store bytes, [(off, type, first-round status, reason)], summary dict), and with a funding table (a
    tests/gossip_store_funding.py Table) also (verdict per row, funding summary).  sigcheck(msg, signer33 or None) gives
    a message's status as for tests/gossip_store.py audit(); None leaves every message status 0.  With a table, rule 2
    also deletes an announcement whose first-round status is 0 and whose verdict is refused (GP_FUNDING)."""
    if store[0] >> 5:
        raise ValueError("major version")
    recs, end, stop, no_amount = walk(store, truncated_stops=False)
    bad = {i for i, (off, typ, ln, st) in enumerate(recs) if st == 0 and not crc_ok(store, off)}
    live = [i for i, r in enumerate(recs) if r[3] == 0 and i not in bad]

    def check(i, h):
        off, ln = recs[i][0], recs[i][2]
        return sigcheck(store[off + HDR:off + HDR + ln], signer(store, recs, i, h)) if sigcheck else 0

    # first round: the audit's statuses over the records with good checksums
    h1 = holders(store, recs, live)
    status = {i: check(i, h1.get(i)) for i in live if recs[i][1] in (256, 257, 258)}
    fund = {} if table is None else {
        i: gf.verdict(store, recs[i][0], table) for i in live if recs[i][1] == 256 and status[i] == 0}
    reason = {i: GP_TRUNCATED for i, r in enumerate(recs) if r[3] == TRUNCATED}
    reason.update({i: GP_BAD_CRC for i in bad})
    for i, st in status.items():
        if (st in (-1, -3)) if recs[i][1] == 258 else st != 0:
            reason[i] = GP_MESSAGE
        elif fund.get(i) in gf.REFUSED:
            reason[i] = GP_FUNDING
    # second round: the table without the deleted announcements
    h2 = holders(store, recs, [i for i in live if not (recs[i][1] == 256 and i in reason)])
    reverified = 0
    for i in live:
        typ = recs[i][1]
        if i in reason:
            continue
        if typ == 256:
            if h2.get(i) is not None:
                reason[i] = GP_REDUNDANT
        elif typ == 258:
            h = h2.get(i)
            if h is None:
                reason[i] = GP_NO_CHANNEL
            elif h != h1.get(i):
                reverified += 1
                if check(i, h) != 0:
                    reason[i] = GP_SIGNATURE
            elif status[i] != 0:
                reason[i] = GP_SIGNATURE
        elif typ not in (257,) + STORE_TYPES:
            reason[i] = GP_UNKNOWN
    # the amount record right after a deleted announcement goes with it
    for i in range(1, len(recs)):
        if recs[i][3] == 0 and i not in reason and recs[i][1] == CHANNEL_AMOUNT and recs[i - 1][1] == 256 and i - 1 in reason:
            reason[i] = GP_AMOUNT
    # an announcement kept without room for its amount record stops the walk
    cut = no_amount if no_amount is not None and no_amount not in reason else len(recs)
    out = bytearray(store)
    rows, fv = [], []
    for i, (off, typ, ln, st) in enumerate(recs):
        if i >= cut:
            st = NO_AMOUNT if i == cut else NOT_REACHED
        elif st == 0:
            st = BAD_CRC if i in bad else status[i] if i in status else (STORE_RECORD if typ in STORE_TYPES else UNKNOWN)
        why = reason.get(i, GP_KEPT) if i < cut else GP_KEPT
        if why:
            out[off] |= DELETED >> 8
        rows.append((off, typ, st, why))
        fv.append(fund.get(i, gf.GF_NONE) if i < cut else gf.GF_NONE)
    whys = [w for _, _, _, w in rows]
    s = dict(version=store[0], stop=NO_AMOUNT if cut < len(recs) else stop,
             end_offset=recs[cut][0] if cut < len(recs) else end, records=len(recs),
             pruned=sum(w != GP_KEPT for w in whys), reverified=reverified)
    for k, name in enumerate(REASONS, GP_BAD_CRC):
        s[name] = whys.count(k)
    if table is None:
        return bytes(out), rows, s
    return bytes(out), rows, s, fv, gf.summary(fv, whys.count(GP_FUNDING))
