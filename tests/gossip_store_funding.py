"""Python model of the funding check of a gossip_store (sv_verify_gossip_store_funding_host and
sv_prune_gossip_store_funding_host, include/cln_sigverify.h): one verdict per channel_announcement from lightningd's
funding outputs, following get_txout (lightningd/gossip_control.c:78-115) and gossipd's txout reply
(gossipd/gossmap_manage.c:696-699, :791-819, :850-852).  Built on the audit's model (tests/gossip_store.py); the
prune with those refused deleted in rule 2 is tests/gossip_store_prune.py prune with a table."""
import hashlib
import struct

from tests import gossip_store as gs
from tests.gossip_store import CHANNEL_AMOUNT, HDR

# verdicts (include/cln_sigverify.h SV_GF_*)
GF_NONE, GF_FUNDED, GF_UNCHECKED, GF_DYING, GF_NO_TXOUT, GF_SCRIPT, GF_AMOUNT = range(7)
REFUSED = (GF_NO_TXOUT, GF_SCRIPT, GF_AMOUNT)
DYING = 0x0800
NAMES = {GF_FUNDED: "funded", GF_UNCHECKED: "unchecked", GF_DYING: "dying", GF_NO_TXOUT: "no_txout",
         GF_SCRIPT: "script", GF_AMOUNT: "amount"}


def redeem_2of2(k1, k2):
    """bitcoin_redeem_2of2 (bitcoin/script.c:151-167): OP_2 <ka> <kb> OP_2 OP_CHECKMULTISIG, keys in memcmp order"""
    a, b = (k1, k2) if k1 < k2 else (k2, k1)
    return bytes([0x52, 33]) + a + bytes([33]) + b + bytes([0x52, 0xAE])


def p2wsh_2of2(k1, k2):
    """scriptpubkey_p2wsh of the 2-of-2: OP_0 PUSH32 SHA-256(script)"""
    return b"\x00\x20" + hashlib.sha256(redeem_2of2(k1, k2)).digest()


def ann_keys(store, p):
    """(scid as u64, bitcoin_key_1, bitcoin_key_2) of the announcement whose message starts at p"""
    f = p + 260 + struct.unpack(">H", store[p + 258:p + 260])[0]
    return struct.unpack(">Q", store[f + 32:f + 40])[0], store[f + 106:f + 139], store[f + 139:f + 172]


class Table:
    """the funding table as dicts: outputs {scid: (satoshis, script34)}, blocks {height}"""

    def __init__(self, outputs, blocks):
        self.outputs = dict(outputs)
        self.blocks = set(blocks)

    @classmethod
    def of(cls, ft):
        """from a lightning_b200.funding.FundingTable"""
        return cls({int(s): (int(a), bytes(c)) for s, a, c in zip(ft.scid, ft.satoshis, ft.script)},
                   [int(b) for b in ft.blocks])


def verdict(store, hdr_off, table):
    """the verdict of the channel_announcement whose record header is at hdr_off"""
    flags, ln = struct.unpack(">HH", store[hdr_off:hdr_off + 4])
    if flags & DYING:
        return GF_DYING
    scid, k1, k2 = ann_keys(store, hdr_off + HDR)
    out = table.outputs.get(scid)
    if out is None:
        return GF_NO_TXOUT if scid >> 40 in table.blocks else GF_UNCHECKED
    sats, script = out
    if script != p2wsh_2of2(k1, k2):
        return GF_SCRIPT
    a = hdr_off + HDR + ln
    if a + HDR + 2 + 8 > len(store) or struct.unpack(">H", store[a + HDR:a + HDR + 2])[0] != CHANNEL_AMOUNT:
        return GF_AMOUNT
    return GF_FUNDED if struct.unpack(">Q", store[a + HDR + 2:a + HDR + 10])[0] == sats else GF_AMOUNT


def summary(verdicts, deleted=0):
    s = dict(checked=sum(v != GF_NONE for v in verdicts), deleted=deleted)
    for v, k in NAMES.items():
        s[k] = sum(x == v for x in verdicts)
    return s


def audit(store, table, sigcheck=None):
    """-> (the audit's rows as tests/gossip_store.py audit gives them, summary, verdict per row, funding summary)"""
    rows, s = gs.audit(store, sigcheck)
    fund = [verdict(store, off, table) if typ == 256 and st == 0 else GF_NONE for off, typ, st, _ in rows]
    return rows, s, fund, summary(fund)


def table_of_store(store):
    """the table that funds every channel of a store as its own amount records say: for each live announcement (first of
    its scid) followed by a channel_amount, an output at its scid with the 2-of-2 script and that amount; every block
    processed.  -> (scid list, satoshis list, scripts list, block list)"""
    recs = gs.walk(store)[0]
    seen = {}
    for i, (off, typ, ln, st) in enumerate(recs):
        if st or typ != 256 or i + 1 >= len(recs) or recs[i + 1][1] != CHANNEL_AMOUNT:
            continue
        scid, k1, k2 = ann_keys(store, off + HDR)
        a = recs[i + 1][0]
        if scid not in seen:
            seen[scid] = (struct.unpack(">Q", store[a + HDR + 2:a + HDR + 10])[0], p2wsh_2of2(k1, k2))
    scids = sorted(seen)
    return scids, [seen[s][0] for s in scids], [seen[s][1] for s in scids], sorted({s >> 40 for s in scids})


# ---- the committed store fixture, funded by a table built from its own announcements, and one mutation per verdict ----
def fixture_cases(fx):
    """name -> (store bytes, (scids, satoshis, scripts, blocks)), from the fixture fx: the table funds every channel as
    its amount records say, then one change per verdict"""
    recs = gs.walk(fx)[0]
    scids, sats, scripts, blocks = table_of_store(fx)
    anns = [i for i, r in enumerate(recs) if r[1] == 256 and r[3] == 0 and i + 1 < len(recs) and recs[i + 1][1] == CHANNEL_AMOUNT]
    pos = {s: k for k, s in enumerate(scids)}

    def scid_of(i):
        return ann_keys(fx, recs[i][0] + HDR)[0]

    def rec(i):
        return fx[recs[i][0]:recs[i][0] + HDR + recs[i][2]]

    def table(drop=(), drop_blocks=(), script=None, sat=None):
        sc, sa, sp = list(scids), list(sats), list(scripts)
        for k, v in (script or {}).items():
            sp[pos[k]] = v
        for k, v in (sat or {}).items():
            sa[pos[k]] = v
        keep = [j for j, s in enumerate(sc) if s not in drop]
        return ([sc[j] for j in keep], [sa[j] for j in keep], [sp[j] for j in keep],
                [b for b in blocks if b not in drop_blocks])

    out = {"clean": (fx, table())}
    s = scid_of(anns[10])
    out["no_txout"] = (fx, table(drop={s}))
    s = scid_of(anns[20])
    out["unchecked"] = (fx, table(drop={s}, drop_blocks={s >> 40}))
    s = scid_of(anns[30])
    _, k1, k2 = ann_keys(fx, recs[anns[30]][0] + HDR)
    lo, hi = sorted((k1, k2))
    out["script_unsorted_keys"] = (fx, table(script={s: b"\x00\x20" + hashlib.sha256(
        bytes([0x52, 33]) + hi + bytes([33]) + lo + bytes([0x52, 0xAE])).digest()}))
    s = scid_of(anns[35])
    _, k1, _ = ann_keys(fx, recs[anns[35]][0] + HDR)
    other = ann_keys(fx, recs[anns[36]][0] + HDR)[2]
    out["script_other_key"] = (fx, table(script={s: p2wsh_2of2(k1, other)}))
    s = scid_of(anns[40])
    out["amount_off_by_one"] = (fx, table(sat={s: sats[pos[s]] + 1}))
    i = anns[50]
    a = recs[i + 1]
    out["amount_record_removed"] = (fx[:a[0]] + fx[a[0] + HDR + a[2]:], table())
    i = anns[55]
    a = recs[i + 1]
    upd = next(j for j, r in enumerate(recs) if r[1] == 258 and r[3] == 0 and
               fx[r[0] + HDR + 98:r[0] + HDR + 106] == struct.pack(">Q", scid_of(i)))
    out["amount_record_replaced"] = (fx[:a[0]] + rec(upd) + fx[a[0] + HDR + a[2]:], table())
    # the dying bit in the header only (the checksum covers the message), with the output spent: still dying, kept
    i = anns[60]
    st = bytearray(fx)
    st[recs[i][0]] |= DYING >> 8
    out["dying"] = (bytes(st), table(drop={scid_of(i)}))
    # the holder's amount record holds one sat more than the output; a correctly funded copy of it follows later with
    # the channel's updates: the copy holds the channel, the updates before it have none
    i = anns[70]
    s = scid_of(i)
    a = recs[i + 1]
    st = bytearray(fx)
    struct.pack_into(">Q", st, a[0] + HDR + 2, sats[pos[s]] + 1)
    gs.reseal(st, a[0])
    mine = [j for j, r in enumerate(recs) if r[1] == 258 and r[3] == 0 and
            fx[r[0] + HDR + 98:r[0] + HDR + 106] == struct.pack(">Q", s)]
    out["refused_holder_then_funded_copy"] = (bytes(st) + rec(i) + rec(i + 1) + b"".join(rec(j) for j in mine), table())
    return out


def corrupt_table(t, rate, seed):
    """(scids, satoshis, scripts, blocks) with about rate of the entries made wrong: the output removed with its block
    kept, the output and its block removed, a script byte flipped, or the amount one sat more"""
    import random
    rng = random.Random(seed)
    sc, sa, sp, bl = list(t[0]), list(t[1]), list(t[2]), set(t[3])
    keep = []
    for j in range(len(sc)):
        if rng.random() >= rate:
            keep.append(j)
            continue
        k = rng.randrange(4)
        if k == 1:
            bl.discard(sc[j] >> 40)
        elif k == 2:
            sp[j] = sp[j][:5] + bytes([sp[j][5] ^ 1]) + sp[j][6:]
            keep.append(j)
        elif k == 3:
            sa[j] += 1
            keep.append(j)
    return [sc[j] for j in keep], [sa[j] for j in keep], [sp[j] for j in keep], sorted(bl)
