"""lightningd's funding outputs, as a gossip_store's channel_announcements are checked against them.

gossipd lets a channel_announcement in only after lightningd answers its txout request (get_txout,
lightningd/gossip_control.c:78-115) from two tables of lightningd.sqlite3:

  utxoset   every P2WSH output of every block lightningd processed, with its spend height; the unspent one at a short
            channel id is what wallet_outpoint_for_scid (wallet/wallet.c:5023-5060) returns
  blocks    the heights lightningd processed (wallet_have_block): no output at a processed height means the announcement
            is refused, an unprocessed height means lightningd would have asked bitcoind

FundingTable holds those two tables as the engine takes them (sv_funding_table, include/cln_sigverify.h).  Read them
with lightningd stopped:

    python -m lightning_b200.funding export ~/.lightning/bitcoin/lightningd.sqlite3 funding.tbl
    cln_verify_gossip_store --funding funding.tbl ~/.lightning/bitcoin/gossip_store

File format (little-endian): the 8 bytes b"CLNFUND1", u64 n_outputs, u64 n_blocks, then n_outputs entries of 50 bytes
[scid u64 | satoshis u64 | scriptpubkey 34 bytes], then n_blocks heights as u32.  scid = block << 40 | txindex << 16 |
outnum.
"""
import argparse
import os
import sqlite3
import struct
import sys

import numpy as np

MAGIC = b"CLNFUND1"
_HEAD = struct.Struct("<8sQQ")
_ENTRY = np.dtype([("scid", "<u8"), ("satoshis", "<u8"), ("script", "u1", (34,))])

# the unspent outputs wallet_outpoint_for_scid finds, and the heights wallet_have_block finds
UTXO_QUERY = "SELECT blockheight, txindex, outnum, scriptpubkey, satoshis FROM utxoset WHERE spendheight IS NULL"
BLOCKS_QUERY = "SELECT height FROM blocks"


def scid(block, txindex, outnum):
    """the short channel id as a u64: block << 40 | txindex << 16 | outnum"""
    if not (0 <= block < 1 << 24 and 0 <= txindex < 1 << 24 and 0 <= outnum < 1 << 16):
        raise ValueError(f"not a short channel id: {block}x{txindex}x{outnum}")
    return block << 40 | txindex << 16 | outnum


class FundingTable:
    """scid (uint64), satoshis (uint64), script (n x 34 uint8) per output, unique scids; blocks (uint32) processed."""

    def __init__(self, scid, satoshis, script, blocks):
        self.scid = np.ascontiguousarray(scid, dtype=np.uint64).reshape(-1)
        self.satoshis = np.ascontiguousarray(satoshis, dtype=np.uint64).reshape(-1)
        self.script = np.ascontiguousarray(script, dtype=np.uint8).reshape(-1, 34)
        self.blocks = np.ascontiguousarray(blocks, dtype=np.uint32).reshape(-1)
        n = self.scid.size
        if self.satoshis.size != n or self.script.shape[0] != n:
            raise ValueError("scid, satoshis and script need one entry per output")
        if np.unique(self.scid).size != n:
            raise ValueError("a short channel id appears twice among the outputs")

    def __len__(self):
        return self.scid.size

    @classmethod
    def from_arrays(cls, scid, satoshis, script, blocks):
        return cls(scid, satoshis, script, blocks)

    @classmethod
    def from_lightningd_db(cls, path):
        """the unspent outputs and processed heights of lightningd.sqlite3 (opened read-only; stop lightningd first)"""
        uri = "file:" + os.path.abspath(path) + "?mode=ro"
        con = sqlite3.connect(uri, uri=True)
        try:
            rows = con.execute(UTXO_QUERY).fetchall()
            heights = [h for (h,) in con.execute(BLOCKS_QUERY)]
        finally:
            con.close()
        scids, sats, scripts = [], [], []
        for block, txindex, outnum, script, sat in rows:
            script = bytes(script)
            if len(script) != 34:
                raise ValueError(f"utxoset {block}x{txindex}x{outnum}: scriptpubkey of {len(script)} bytes, not 34 (P2WSH)")
            scids.append(scid(block, txindex, outnum))
            sats.append(sat)
            scripts.append(np.frombuffer(script, np.uint8))
        return cls(np.array(scids, np.uint64), np.array(sats, np.uint64),
                   np.array(scripts, np.uint8).reshape(-1, 34), np.array(heights, np.uint32))

    def to_bytes(self):
        e = np.zeros(len(self), _ENTRY)
        e["scid"], e["satoshis"], e["script"] = self.scid, self.satoshis, self.script
        return _HEAD.pack(MAGIC, len(self), self.blocks.size) + e.tobytes() + self.blocks.astype("<u4").tobytes()

    @classmethod
    def from_bytes(cls, data):
        if len(data) < _HEAD.size or data[:8] != MAGIC:
            raise ValueError("not a funding table (bad magic)")
        _, n, nb = _HEAD.unpack_from(data)
        if len(data) != _HEAD.size + n * _ENTRY.itemsize + 4 * nb:
            raise ValueError(f"funding table of {len(data)} bytes does not hold {n} outputs and {nb} heights")
        e = np.frombuffer(data, _ENTRY, n, _HEAD.size)
        blocks = np.frombuffer(data, "<u4", nb, _HEAD.size + n * _ENTRY.itemsize)
        return cls(e["scid"], e["satoshis"], e["script"], blocks)

    def save(self, path):
        with open(path, "wb") as f:
            f.write(self.to_bytes())

    @classmethod
    def load(cls, path):
        with open(path, "rb") as f:
            return cls.from_bytes(f.read())


def main(argv=None):
    ap = argparse.ArgumentParser(prog="python -m lightning_b200.funding",
                                 description="export lightningd's funding outputs for cln_verify_gossip_store --funding")
    sub = ap.add_subparsers(dest="cmd", required=True)
    ex = sub.add_parser("export", help="read lightningd.sqlite3 (lightningd stopped), write the table file")
    ex.add_argument("db")
    ex.add_argument("out")
    a = ap.parse_args(argv)
    t = FundingTable.from_lightningd_db(a.db)
    t.save(a.out)
    print(f"{a.out}: {len(t)} unspent outputs, {t.blocks.size} processed blocks")
    return 0


if __name__ == "__main__":
    sys.exit(main())
