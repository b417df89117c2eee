#!/usr/bin/env python3
"""Generate tests/golden/gossip_store_subset.bin/.json from the reference tree (run where CLN_SRC names a Core Lightning
source tree; the GPU box only sees the generated files).

  gossip_store_subset.bin/.json   the records of tests/data/routing_gossip_store that hold the messages of
                                  gossip_subset.bin (make_golden.py), each channel_announcement with the channel_amount
                                  record after it, copied verbatim (CLN's own headers and checksums) in store order
                                  behind the store's version byte: a small store gossmap loads as it is.

Every checksum of the source store is re-checked with tests/gossip_store.py's CRC-32C before anything is copied.
"""
import json
import os
import struct
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from tests import gossip_store as gs  # noqa: E402

REF = os.environ["CLN_SRC"]  # a Core Lightning source tree
OUT = os.path.dirname(os.path.abspath(__file__))
WIRE_CHANNEL_ANNOUNCEMENT, WIRE_CHANNEL_UPDATE = 256, 258


def gossip_store_subset():
    data = open(REF + "/tests/data/routing_gossip_store", "rb").read()
    recs, _, stop, _ = gs.walk(data)
    assert stop == gs.EOF and all(st == 0 and gs.crc_ok(data, off) for off, _, _, st in recs)
    want = open(OUT + "/gossip_subset.bin", "rb").read()
    msgs, pos = [], 0
    while pos < len(want):
        (ln,) = struct.unpack(">H", want[pos:pos + 2])
        msgs.append(want[pos + 2:pos + 2 + ln])
        pos += 2 + ln
    out, k = [data[:1]], 0
    for i, (off, typ, ln, _) in enumerate(recs):
        if k < len(msgs) and data[off + 12:off + 12 + ln] == msgs[k]:
            out.append(data[off:off + 12 + ln])
            if typ == WIRE_CHANNEL_ANNOUNCEMENT:
                aoff, atyp, aln, _ = recs[i + 1]
                assert atyp == gs.CHANNEL_AMOUNT
                out.append(data[aoff:aoff + 12 + aln])
            k += 1
    assert k == len(msgs), (k, len(msgs))
    blob = b"".join(out)
    sub, _ = gs.audit(blob)
    assert all(st in (0, gs.STORE_RECORD) for _, _, st, _ in sub)
    assert all(h is not None for _, t, _, h in sub if t == WIRE_CHANNEL_UPDATE)
    open(OUT + "/gossip_store_subset.bin", "wb").write(blob)
    json.dump(dict(source="tests/data/routing_gossip_store (reference v26.04.1)",
                   format="gossip_store: version byte, then records (be16 flags, be16 len, be32 crc32c, be32 timestamp, message)",
                   version=blob[0], records=len(sub), bytes=len(blob), messages=len(msgs),
                   channel_announcements=sum(t == 256 for _, t, _, _ in sub), node_announcements=sum(t == 257 for _, t, _, _ in sub),
                   channel_updates=sum(t == 258 for _, t, _, _ in sub), channel_amounts=sum(t == gs.CHANNEL_AMOUNT for _, t, _, _ in sub)),
              open(OUT + "/gossip_store_subset.json", "w"), indent=1)
    print("gossip_store subset:", len(sub), "records,", len(blob), "bytes")


if __name__ == "__main__":
    gossip_store_subset()
