"""Funding tables shaped as lightningd exports them, for the funding check of a gossip_store
(tests/gossip_store_funding.py is its model).  FundingTable.from_lightningd_db keeps utxoset's rows in the order SQLite
returns them, so the engine's sort is the only thing that orders a real table; and utxoset holds every unspent P2WSH
output of every processed block, so a real table is large and full of outputs no announcement of the store names.

A table here is four numpy arrays (scid u64[n], satoshis u64[n], script u8[n, 34], blocks u32[m]); arrays() takes the
(scids, satoshis, scripts, blocks) lists of tests/gossip_store_funding.py too.  Everything is seeded.

  ORDERS      the outputs and the heights each put in another order: reversed, shuffled, low bits first, and shuffled
              with every height listed twice
  decoys()    outputs that fund no announcement: each announced scid's neighbours (txindex, outnum and block +-1), its
              64 single-bit flips (for a sample), 0, 1, 2^64-1, block 2^24-1, uniform scids; each with the script and
              amount of a real entry, some amounts >= 2^63
  pad()       a table of exactly n outputs and m heights: the real entries (a seeded subset when n is smaller), then
              decoys; heights no announcement lies in
  SIZES       output counts on both sides of the CUB radix sort's single-tile limit and its onesweep tile, 2^16 +-1,
              2^20 +-1 and 2^22
  features_store()  a signed store whose announcements carry features fields of many lengths, with a table that gives
              each one every verdict"""
import functools
import hashlib
import struct

import numpy as np

from tests import ecc
from tests import gossip_store as gs
from tests import gossip_store_funding as gf

ORDERS = ("reversed", "shuffled", "low_bits_first", "shuffled_heights_twice")
# cub::DeviceRadixSort on sm_90 (CUDA 12.9, Policy900): one tile of SingleTilePolicy holds 256 x 19 items of 4 bytes,
# scaled to the dominant type: 2,304 outputs (8-byte scids), 4,864 heights; above that the onesweep kernels run, with
# 384 x 15 = 5,760 outputs per tile
TILE_OUT, TILE_BLK, ONESWEEP_OUT = 2304, 4864, 5760
SIZES = (2000, TILE_OUT - 1, TILE_OUT, TILE_OUT + 1, 3000, TILE_BLK - 1, TILE_BLK, TILE_BLK + 1, 5000, ONESWEEP_OUT,
         ONESWEEP_OUT + 1, (1 << 16) - 1, (1 << 16) + 1, (1 << 20) - 1, (1 << 20) + 1, 1 << 22)
BIG = 1 << 22


def _unique(x):
    """np.unique by sorting (numpy's hash-based unique is several times slower on millions of keys)"""
    x = np.sort(x)
    return x[np.concatenate([[True], x[1:] != x[:-1]])] if x.size else x


def arrays(t):
    """(scid u64, satoshis u64, script u8 (n, 34), blocks u32) of a table given as arrays or as lists"""
    sc, sa, sp, bl = t
    sc = np.array(sc, np.uint64).reshape(-1)
    if isinstance(sp, np.ndarray):
        sp = sp.reshape(-1, 34).astype(np.uint8)
    else:
        sp = np.frombuffer(b"".join(sp), np.uint8).reshape(-1, 34) if len(sp) else np.zeros((0, 34), np.uint8)
    return sc, np.array(sa, np.uint64).reshape(-1), np.ascontiguousarray(sp), np.array(bl, np.uint32).reshape(-1)


def take(a, idx, blocks=None):
    """the outputs at idx (in that order), and blocks (the table's own when None)"""
    return a[0][idx], a[1][idx], a[2][idx], a[3] if blocks is None else blocks


def reorder(a, order, seed):
    """the table with its outputs and its heights each put in `order` (one of ORDERS)"""
    rng = np.random.default_rng(seed)
    sc, bl = a[0], a[3]
    if order == "reversed":
        return take(a, np.arange(sc.size)[::-1], bl[::-1].copy())
    if order == "shuffled":
        return take(a, rng.permutation(sc.size), bl[rng.permutation(bl.size)])
    if order == "low_bits_first":
        # sorted by (outnum, txindex, block), the heights by (low 16 bits, high 16 bits): what a sort that reads only
        # the low bits leaves in place
        idx = np.lexsort((sc >> np.uint64(40), (sc >> np.uint64(16)) & np.uint64(0xFFFFFF), sc & np.uint64(0xFFFF)))
        return take(a, idx, bl[np.lexsort((bl >> np.uint32(16), bl & np.uint32(0xFFFF)))])
    if order == "shuffled_heights_twice":
        twice = np.concatenate([bl, bl])
        return take(a, rng.permutation(sc.size), twice[rng.permutation(twice.size)])
    raise ValueError(order)


def sort(a):
    """the table with its outputs sorted by scid and its heights sorted (as the engine's sorts leave them)"""
    return take(a, np.argsort(a[0], kind="stable"), np.sort(a[3]))


def announced(store):
    """the scids (u64 array) of every channel_announcement the walk of store reaches, whatever its status"""
    out = set()
    for off, typ, ln, st in gs.walk(store)[0]:
        p = off + gs.HDR
        if typ == 256 and gs.ann_ok(store, p):
            out.add(gf.ann_keys(store, p)[0])
    return np.array(sorted(out), np.uint64)


def _fields(s):
    return s >> np.uint64(40), (s >> np.uint64(16)) & np.uint64(0xFFFFFF), s & np.uint64(0xFFFF)


def neighbours(ann):
    """for each announced scid: txindex +-1, outnum +-1 and block +-1 with the other fields kept (where they stay in
    their range)"""
    blk, tx, out = _fields(ann)
    one = np.uint64(1)
    parts = []
    for d, field, top in ((one << np.uint64(16), tx, (1 << 24) - 1), (one, out, (1 << 16) - 1),
                          (one << np.uint64(40), blk, (1 << 24) - 1)):
        parts += [ann[field < np.uint64(top)] + d, ann[field > np.uint64(0)] - d]
    return np.concatenate(parts) if parts else np.zeros(0, np.uint64)


def bit_flips(ann):
    """every scid of ann with exactly one of its 64 bits flipped: keys that differ from an announced one in one radix
    digit only"""
    bits = np.uint64(1) << np.arange(64, dtype=np.uint64)
    return (ann[:, None] ^ bits[None, :]).reshape(-1)


SPECIAL = np.array([0, 1, (1 << 64) - 1, ((1 << 24) - 1) << 40, ((1 << 24) - 1) << 40 | 1], np.uint64)


def decoys(a, ann, count, seed, flips=64):
    """count outputs (fewer only when count is smaller than the structured set; then a seeded sample of it) that
    fund no announcement: neighbours of every announced scid, the single-bit flips of `flips` announced scids, SPECIAL,
    then seeded uniform scids.  Each carries the script and amount of a real entry of a (amounts of every 5th with bit
    63 set).  -> (scid, satoshis, script)"""
    rng = np.random.default_rng(seed)
    ann = np.asarray(ann, np.uint64)
    pick = ann[rng.permutation(ann.size)[:flips]]
    cand = _unique(np.concatenate([neighbours(ann), bit_flips(pick), SPECIAL]))
    cand = cand[~np.isin(cand, ann) & ~np.isin(cand, a[0])]
    cand = cand[rng.permutation(cand.size)][:count]
    while cand.size < count:
        more = _unique(rng.integers(0, 1 << 64, 2 * (count - cand.size) + 64, dtype=np.uint64))
        more = more[~np.isin(more, ann) & ~np.isin(more, a[0]) & ~np.isin(more, cand)]
        cand = np.concatenate([cand, more[rng.permutation(more.size)][:count - cand.size]])
    assert not np.isin(cand, ann).any(), "a decoy equals an announced scid"
    assert _unique(cand).size == cand.size
    src = rng.integers(0, a[0].size, cand.size)
    sats = a[1][src].copy()
    sats[::5] |= np.uint64(1) << np.uint64(63)
    return cand, sats, a[2][src].copy()


def decoy_heights(ann, count, seed):
    """count distinct heights no announced scid lies in: the announced blocks +-1 and their single-bit flips, 0,
    2^32-1, 2^24-1, then uniform"""
    rng = np.random.default_rng(seed)
    used = _unique((np.asarray(ann, np.uint64) >> np.uint64(40)).astype(np.uint32))
    bits = np.uint32(1) << np.arange(32, dtype=np.uint32)
    cand = _unique(np.concatenate([used + np.uint32(1), used - np.uint32(1), (used[:16, None] ^ bits[None, :]).reshape(-1),
                                     np.array([0, 0xFFFFFFFF, (1 << 24) - 1], np.uint32)]))
    cand = cand[~np.isin(cand, used)]
    cand = cand[rng.permutation(cand.size)][:count]
    if cand.size < count:
        more = _unique(rng.integers(0, 1 << 32, 2 * count + 64, dtype=np.uint64).astype(np.uint32))
        more = more[~np.isin(more, used) & ~np.isin(more, cand)]
        cand = np.concatenate([cand, more[rng.permutation(more.size)][:count - cand.size]])
    assert cand.size == count and not np.isin(cand, used).any()
    return cand


def pad(a, ann, n, m, seed):
    """a table of exactly n outputs and m heights, seeded: when n is below a's size, a seeded subset of a's outputs,
    else all of them and n - len decoys; a's heights, then (when m is larger) decoy heights, or a seeded subset of
    a's heights when m is smaller.  The outputs come in a seeded shuffle."""
    rng = np.random.default_rng(seed)
    k = a[0].size
    if n <= k:
        out = take(a, np.sort(rng.permutation(k)[:n]))
    else:
        d = decoys(a, ann, n - k, seed + 1)
        out = (np.concatenate([a[0], d[0]]), np.concatenate([a[1], d[1]]), np.concatenate([a[2], d[2]]), a[3])
    bl = a[3]
    bl = bl[np.sort(rng.permutation(bl.size)[:m])] if m <= bl.size else np.concatenate(
        [bl, decoy_heights(ann, m - bl.size, seed + 2)])
    p = rng.permutation(out[0].size)
    return out[0][p], out[1][p], out[2][p], bl


def model(a, ann):
    """the model's table (gf.Table) of a, holding only the outputs at announced scids and the heights of announced
    blocks: the verdicts read no others, so this is exact for every store whose announced scids are ann, and it stays
    small for a table of millions"""
    ann = np.asarray(ann, np.uint64)
    keep = np.isin(a[0], ann)
    sc, sa, sp = a[0][keep], a[1][keep], a[2][keep]
    bl = _unique(a[3])
    bl = bl[np.isin(bl, (ann >> np.uint64(40)).astype(np.uint32))]
    return gf.Table({int(s): (int(x), sp[i].tobytes()) for i, (s, x) in enumerate(zip(sc, sa))}, (int(b) for b in bl))


def same_model(a, b, ann):
    """a and b give the same model: the same outputs at announced scids and the same processed announced blocks"""
    ta, tb = model(a, ann), model(b, ann)
    return ta.outputs == tb.outputs and ta.blocks == tb.blocks


def lists(a):
    """the (scids, satoshis, scripts, blocks) lists of tests/gossip_store_funding.py"""
    return [int(x) for x in a[0]], [int(x) for x in a[1]], [x.tobytes() for x in a[2]], [int(x) for x in a[3]]


# ---- a signed store whose announcements carry features ---------------------------------------------------------------
FLENS = (0, 1, 2, 7, 8, 33, 255, 256, 1000)
KINDS = ("funded", "script", "amount", "no_txout", "unchecked")
_SK = {n: hashlib.sha256(n.encode()).digest() for n in ("fa", "fb", "fba", "fbb", "fbx")}
_PUB = {n: ecc.pubkey_create(sk)[0] for n, sk in _SK.items()}
TESTNET = bytes.fromhex("43497fd7f826957108f4a30fd9cec3aeba79972084e90ead01ea330900000000")


def _sha256d(b):
    return hashlib.sha256(hashlib.sha256(b).digest()).digest()


def make_ca(scid, features, n1="fa", n2="fb", b1="fba", b2="fbb", chain=TESTNET):
    """a channel_announcement signed by all four keys, with `features` as its features field (node ids in order)"""
    if _PUB[n1] > _PUB[n2]:
        n1, n2 = n2, n1
    tail = struct.pack(">H", len(features)) + features + chain + struct.pack(">Q", scid) + _PUB[n1] + _PUB[n2] + \
        _PUB[b1] + _PUB[b2]
    h = _sha256d(tail)
    return b"\x01\x00" + b"".join(ecc.ecdsa_sign(_SK[k], h) for k in (n1, n2, b1, b2)) + tail


def scid_of(block, txindex, outnum):
    return block << 40 | txindex << 16 | outnum


@functools.lru_cache(maxsize=None)
def features_store():
    """-> (store, table as arrays, {scid: (flen, kind)}).  For every features length of FLENS and every verdict of
    KINDS, one signed announcement followed by its channel_amount, and the table entry (or its absence, or its
    block's) that gives it that verdict.  Amounts of the funded ones with bit 63 set at odd flen indices.  Where the
    features field reaches past the bitcoin keys (172 bytes), the bytes a read that ignores its length would take for
    the scid and the keys are the scid and keys of the funded announcement with flen 0, whose output holds this
    announcement's amount: such a read would then find a funded output where there is none, or the wrong one."""
    rng = np.random.default_rng(4101)
    keys = _PUB["fba"], _PUB["fbb"]
    good = gf.p2wsh_2of2(*keys)
    recs, sc, sa, sp, blocks, what = [], [], [], [], [], {}
    decoy_scid = scid_of(2_000_000, 1, 0)  # the funded, flen 0 announcement: every long features field names it
    decoy_amt = int(rng.integers(1000, 1 << 40))
    for i, flen in enumerate(FLENS):
        for j, kind in enumerate(KINDS):
            s = scid_of(2_000_000 + 10 * i + j, 1 + j, i)
            what[s] = (flen, kind)
            amt = decoy_amt if s == decoy_scid or flen >= 172 else \
                int(rng.integers(1000, 1 << 40)) | ((1 << 63) if (i & 1 and kind == "funded") else 0)
            feat = bytearray(rng.integers(0, 256, flen, dtype=np.uint8).tobytes())
            if flen >= 172:
                feat[32:40] = struct.pack(">Q", decoy_scid)
                feat[106:139], feat[139:172] = keys
            recs.append(gs.record(make_ca(s, bytes(feat))))
            recs.append(gs.record(struct.pack(">HQ", gs.CHANNEL_AMOUNT, amt)))
            if kind != "unchecked":
                blocks.append(s >> 40)
            if kind in ("funded", "script", "amount"):
                sc.append(s)
                sa.append(amt + (1 if kind == "amount" else 0))
                sp.append(good if kind != "script" else gf.p2wsh_2of2(keys[0], _PUB["fbx"]))
    store = bytes([16]) + b"".join(recs)
    return store, arrays((sc, sa, sp, blocks)), what
