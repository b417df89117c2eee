"""GPU: no item changes another item's verdict, on every verification route.

The special items of tests/isolation.py go into 64 blocks of 64 items, block b holding the special at offset b, among a
valid background and one with about 25 % flipped messages (device generator, verdicts known by construction).  One batch
so puts a special at every offset of the prep kernel's 32-signature inversion, of the final kernels' 16-item inversions,
of a small-batch CTA and its lane pairs, and in all 8 warps of a throughput CTA.  Every case checks the whole verdict
vector and names the route it must take through the launch counter (tests/test_gpu_routes.py).  Ragged tails, two
specials of different classes in one 16-item unit, whole 32-item units of one special, a seeded permutation, BIP-340
batch verification with specials inside its 1024-signature groups, and gossip batches whose keys collide in the
de-duplication table."""
import hashlib

import numpy as np
import pytest

from tests import ecc
from tests import isolation as I
from tests.test_gpu_routes import KEYLEN, LAUNCHES, counted, main_route
from tests.test_isolation_emul import samekey_batch, samekey_specials

pytestmark = pytest.mark.gpu
BLOCKS = SIZE = 64
N_ITEMS = BLOCKS * SIZE
POS = I.block_positions(BLOCKS, SIZE)
# the routes each kind's block layouts take, checked for complete coverage at the end
ROUTES = {0: ["main_ns", "main_plain", "small", "device", "mixed", "flush", "samekey"],
          1: ["main_ns", "small", "device", "mixed", "flush", "samekey"],
          2: ["main_ns", "main_plain", "small_ns", "small_plain", "device", "mixed", "flush"]}
COVERAGE = I.Coverage()


@pytest.fixture()
def defaults(engine):
    sm = engine.small_max()
    yield sm
    engine.set_small_max(sm)
    engine.set_nosqrt(True)


@pytest.fixture(scope="module")
def backgrounds(engine):
    """{(kind, name): (msg, key, sig, want)} of N_ITEMS + 31 device-generated items, valid or with flipped messages"""
    import torch
    out = {}
    n = N_ITEMS + 31
    for kind in (0, 1, 2):
        msg = torch.empty((n, 32), dtype=torch.uint8, device="cuda")
        key = torch.empty((n, KEYLEN[kind]), dtype=torch.uint8, device="cuda")
        sig = torch.empty((n, 64), dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        engine.synth_device(kind, 8100 + kind, n, msg.data_ptr(), key.data_ptr(), sig.data_ptr())
        engine.sync()
        bg = tuple(t.cpu().numpy() for t in (msg, key, sig)) + (np.ones(n, np.uint8),)
        out[(kind, "valid")] = bg
        out[(kind, "flipped")] = I.with_flips(bg, 8200 + kind)
    return out


def check(got, want, placed, what, unit=SIZE):
    bad = I.mismatch(got, want, placed, unit)
    assert bad is None, f"{what}\n{bad}"


def _mixed(kind, batch, backgrounds, name):
    """the kind's batch interleaved item by item with background items of the two other kinds: (kinds, msg, key64,
    sig, want, where the kind's items sit)"""
    n = batch[0].shape[0]
    kinds = np.tile(np.array([0, 1, 2], np.uint8), n)
    msg = np.zeros((3 * n, 32), np.uint8)
    key = np.full((3 * n, 64), 0xEE, np.uint8)
    sig = np.zeros((3 * n, 64), np.uint8)
    want = np.zeros(3 * n, np.uint8)
    for k in (0, 1, 2):
        m, q, s, w = batch if k == kind else (a[:n] for a in backgrounds[(k, name)])
        sl = slice(k, 3 * n, 3)
        msg[sl], sig[sl], want[sl] = m, s, w
        key[sl, :KEYLEN[k]] = q
    return kinds, msg, key, sig, want, np.arange(n) * 3 + kind


def test_block_layout_every_route(engine, backgrounds, defaults):
    """every special at every offset of a 64-item block, both backgrounds: throughput kernels with and without the square
    root, small-batch kernel, sv_verify_device with a bitmap, an interleaved mixed batch, and the deferral queue"""
    import torch
    sm = defaults
    for kind in (0, 1, 2):
        for sp in I.catalogue(kind):
            placed = {int(p): sp for p in POS}
            for name in ("valid", "flipped"):
                msg, key, sig, want = I.block_layout(backgrounds[(kind, name)], sp, BLOCKS, SIZE)
                tag = f"kind {kind} {name} background, {sp.label}"
                engine.set_small_max(0)
                for nosqrt in ((True, False) if kind != 1 else (True,)):
                    engine.set_nosqrt(nosqrt)
                    got = counted(engine, lambda: engine.verify(kind, msg, key, sig), main_route(kind, nosqrt))
                    check(got, want, placed, f"{tag}: throughput kernels, nosqrt {nosqrt}")
                    COVERAGE.add("main_ns" if nosqrt else "main_plain", sp, POS)
                engine.set_small_max(sm)
                for nosqrt in ((True, False) if kind == 2 else (True,)):
                    engine.set_nosqrt(nosqrt)
                    got = counted(engine, lambda: engine.verify(kind, msg, key, sig), "small")
                    check(got, want, placed, f"{tag}: small-batch kernel, nosqrt {nosqrt}")
                    COVERAGE.add("small" if kind != 2 else ("small_ns" if nosqrt else "small_plain"), sp, POS)
                engine.set_nosqrt(True)
                # on the device with the verdict bitmap, throughput kernels
                engine.set_small_max(0)
                d = [torch.from_numpy(a).cuda() for a in (msg, key, sig)]
                out = torch.zeros(N_ITEMS, dtype=torch.uint8, device="cuda")
                bm = torch.zeros(N_ITEMS // 32, dtype=torch.int32, device="cuda")
                torch.cuda.synchronize()
                counted(engine, lambda: engine.verify_device(kind, d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), N_ITEMS,
                                                             out.data_ptr(), bm.data_ptr()), main_route(kind, True), "bitmap")
                engine.sync()
                check(out.cpu().numpy(), want, placed, f"{tag}: sv_verify_device")
                bits = np.unpackbits(bm.cpu().numpy().view(np.uint8), bitorder="little")
                check(bits, want, placed, f"{tag}: verdict bitmap")
                COVERAGE.add("device", sp, POS)
                # interleaved with the two other kinds: the special's neighbours in the batch are items of other kinds
                kinds, m3, k3, s3, w3, at = _mixed(kind, (msg, key, sig, want), backgrounds, name)
                got = counted(engine, lambda: engine.verify_mixed(kinds, m3, k3, s3), "mixed_split",
                              *[r for k in (0, 1, 2) for r in ("mixed_kind", main_route(k, True))])
                check(got[at], want, placed, f"{tag}: mixed batch, the kind's items")
                assert np.array_equal(got, w3), (tag, "mixed batch, the other kinds' items")
                COVERAGE.add("mixed", sp, POS)
                if name == "valid":
                    for i in range(N_ITEMS):
                        engine.enqueue(kind, msg[i], key[i], sig[i])
                    got = counted(engine, engine.flush, main_route(kind, True))
                    check(got, want, placed, f"{tag}: enqueue / flush")
                    COVERAGE.add("flush", sp, POS)
                engine.set_small_max(sm)
    missing = COVERAGE.missing({k: [r for r in ROUTES[k] if r != "samekey"] for k in ROUTES},
                               {k: I.catalogue(k) for k in ROUTES}, range(SIZE))
    assert not missing, missing[:10]
    # every final-batch route (k_final_ecdsa33, k_final_schnorr_ns, k_final_schnorr) had specials handed to the plain path
    # and specials rejected before the curve work beside pending neighbours in their 16-item unit
    for kind, route in ((0, "main_ns"), (2, "main_ns"), (2, "main_plain")):
        classes = {sp.cls for sp in I.catalogue(kind) if len(COVERAGE.seen.get((route, kind, sp.label), ())) == SIZE}
        assert {"exact", "parse"} <= classes, (kind, route, classes)


def test_shared_key_kernel(engine, defaults):
    """sv_verify_samekey_host on the shared-key kernel: each ECDSA special among signatures by its own key"""
    engine.set_small_max(0)
    for kind in (0, 1):
        specials = samekey_specials(kind, I.catalogue(kind))
        assert all(sp.label.startswith("edge.") for sp in I.catalogue(kind) if sp not in specials)
        for sp in specials:
            key, msg, sig, want = samekey_batch(sp, N_ITEMS, BLOCKS, SIZE, 8300 + kind)
            got = counted(engine, lambda: engine.verify_samekey(kind, key, msg, sig), "samekey_shared")
            check(got, want, {int(p): sp for p in POS}, f"kind {kind} shared key: {sp.label}")
            COVERAGE.add("samekey", sp, POS)
        assert not COVERAGE.missing({kind: ["samekey"]}, {kind: specials}, range(SIZE))


def test_tails_pairs_full_units_and_permutation(engine, backgrounds, defaults):
    """the special as the last item of n = 4096 + r (r = 1, 15, 17, 31); two specials of different classes in every
    16-item unit; 32-item units made of one special; and those batches shuffled: verdicts follow the items"""
    sm = defaults
    for kind in (0, 1, 2):
        specials = I.catalogue(kind)
        bg = backgrounds[(kind, "flipped")]
        settings = [(0, True), (0, False), (sm, True)] if kind != 1 else [(0, True), (sm, True)]
        for small_max, nosqrt in settings:
            engine.set_small_max(small_max)
            engine.set_nosqrt(nosqrt)
            for r in (1, 15, 17, 31):
                n = N_ITEMS + r
                for sp in specials:
                    msg, key, sig, want = I.place(bg, n, {n - 1: sp})
                    got = counted(engine, lambda: engine.verify(kind, msg, key, sig),
                                  "small" if n <= small_max else main_route(kind, nosqrt))
                    check(got, want, {n - 1: sp}, f"kind {kind} tail r = {r} small_max {small_max} nosqrt {nosqrt}", 16)
            layouts = [("pairs", N_ITEMS, I.pair_layout(specials, N_ITEMS, 8400 + kind))]
            layouts.append(("full units",) + I.full_unit_layout(specials))
            for name, n, placed in layouts:
                msg, key, sig, want = I.place(backgrounds[(kind, "flipped")], n, placed) if n <= N_ITEMS + 31 else \
                    I.place(tuple(np.concatenate([a] * (n // a.shape[0] + 1)) for a in bg), n, placed)
                route = "small" if n <= small_max else main_route(kind, nosqrt)
                got = counted(engine, lambda: engine.verify(kind, msg, key, sig), route)
                check(got, want, placed, f"kind {kind} {name} small_max {small_max} nosqrt {nosqrt}", 32)
                perm = np.random.default_rng(8500 + kind).permutation(n)
                got2 = counted(engine, lambda: engine.verify(kind, msg[perm], key[perm], sig[perm]), route)
                assert np.array_equal(got2, got[perm]), (kind, name, small_max, nosqrt, "permuted")


def test_bip340_batch_groups_with_specials(engine, backgrounds):
    """BIP-340 batch verification, 4 groups of 1024: each special at every block offset.  Valid specials leave every group
    holding; an item that fails the encoding check drops out without a fallback; any other invalid one fails the groups
    that hold it and only those, and the fallback gives every verdict."""
    seed = bytes(range(32))
    bg = backgrounds[(2, "valid")]
    for sp in I.catalogue(2):
        placed = {int(p): sp for p in POS}
        msg, key, sig, want = I.block_layout(bg, sp, BLOCKS, SIZE)
        holds = sp.want == 1 or not sp.sb_encoding
        routes = ["sb_batch"] if holds else ["sb_batch", "sb_fallback", "small"]
        v, gt, gf = counted(engine, lambda: engine.verify_schnorr_batch(msg, key, sig, seed32=seed), *routes)
        check(v, want, placed, f"batch verification: {sp.label}")
        assert (gt, gf) == (4, 0 if holds else 4), (sp.label, gt, gf)
        if not holds:
            # one copy in group 2 only: that group fails, the three others hold
            pos = 2 * 1024 + 517
            msg, key, sig, want = I.place(bg, N_ITEMS, {pos: sp})
            v, gt, gf = counted(engine, lambda: engine.verify_schnorr_batch(msg, key, sig, seed32=seed), *routes)
            check(v, want, {pos: sp}, f"batch verification, one copy: {sp.label}")
            assert (gt, gf) == (4, 1), (sp.label, gt, gf)
    assert any(sp.want for sp in I.catalogue(2)) and any(not sp.sb_encoding for sp in I.catalogue(2))


# ---- key de-duplication --------------------------------------------------------------------------------------------------
CHAIN = bytes(range(32))


def _update(sk, j):
    """a channel_update signed with sk (tests/ecc.py)"""
    tail = CHAIN + j.to_bytes(8, "big") + (1).to_bytes(4, "big") + b"\x01\x00" + (6).to_bytes(2, "big") + bytes(8) + \
        (1000).to_bytes(4, "big") + (1).to_bytes(4, "big") + (10 ** 9).to_bytes(8, "big")
    return b"\x01\x02" + ecc.ecdsa_sign(sk, hashlib.sha256(hashlib.sha256(tail).digest()).digest()) + tail


def _home_slot(key, mask):
    """the slot k_dedup_insert starts probing from: FNV-1a over the first 12 key bytes"""
    h = 2166136261
    for b in key[:12]:
        h = ((h ^ b) * 16777619) & 0xFFFFFFFF
    return (h ^ (h >> 15)) & mask


# secret keys sha256("isolation/dedup") mod n + offset whose 02||x and 03||x start probing from the same slot of a
# 32768-slot table (the table of small_max + 4096 items at the default small_max): the first such key with y even and
# with y odd, found by walking consecutive keys from the seeded start (about 2^17 point additions, too slow to repeat here)
COLLIDING_OFFSETS = {0: 197178, 1: 42921}


def _colliding_signers(mask):
    """{parity of y: (sk, pub33)} of the keys above; both start probing at the same slot whichever of the two is
    inserted first, so the second compares its full bytes with the other's"""
    out = {}
    for parity, off in COLLIDING_OFFSETS.items():
        sk = (_h_int(b"isolation/dedup") + off).to_bytes(32, "big")
        pub33, _ = ecc.pubkey_create(sk)
        assert pub33[0] == 2 + parity
        x = pub33[1:]
        assert _home_slot(b"\x02" + x, mask) == _home_slot(b"\x03" + x, mask), (parity, mask)
        out[parity] = sk, pub33
    return out


def _h_int(tag):
    return int.from_bytes(hashlib.sha256(tag).digest(), "big") % ecc.N


# launches of one sv_verify_gossip_host call of channel_updates besides the verification itself: k_gossip_slice,
# k_sha256d, k_gossip_status; and the key search when de-duplication is on: k_dedup_insert/number/resolve
GOSSIP_LAUNCHES, DEDUP_SEARCH = 3, 3


def _gossip_both(engine, msgs, signers, want, distinct, uses_dedup):
    """statuses with de-duplication on and off; both equal want.  With it on, the table's distinct key count is what
    the batch holds, and the launch counter pins the path the engine took: the shared tables (k_prep_inv, k_prep_finish,
    k_sharedkey_build_many, k_main_shared) or, past the 40 % repeat threshold, the throughput kernels.  Without the
    square root those two paths launch equally many kernels, so the check runs with it too."""
    n = len(msgs)
    sg = np.frombuffer(b"".join(signers), np.uint8).reshape(n, 33)
    try:
        engine.set_dedup(True)
        for nosqrt in (False, True):
            engine.set_nosqrt(nosqrt)
            path = "samekey_shared" if uses_dedup else main_route(0, nosqrt)
            before = engine.info()["launches"]
            on = engine.verify_gossip(msgs, sg)
            got = engine.info()["launches"] - before
            assert got == GOSSIP_LAUNCHES + DEDUP_SEARCH + LAUNCHES[path], (nosqrt, path, got)
            assert engine.last_distinct_keys() == distinct, (engine.last_distinct_keys(), distinct)
            assert np.array_equal(on, want), ("dedup on", nosqrt, np.nonzero(on != want)[0][:10])
        engine.set_dedup(False)
        before = engine.info()["launches"]
        off = engine.verify_gossip(msgs, sg)
        assert engine.info()["launches"] - before == GOSSIP_LAUNCHES + LAUNCHES[main_route(0, True)]
    finally:
        engine.set_dedup(True)
        engine.set_nosqrt(True)
    assert np.array_equal(off, want), ("dedup off", np.nonzero(off != want)[0][:10])


def test_key_dedup_under_collisions(engine):
    """sv_verify_gossip_host with channel_updates whose listed signers: 02||x next to 03||x (keys chosen so that both
    start probing the table at the same slot: the full-key compare must tell them apart), one undecodable key
    repeated across hundreds of messages, 200+ made-up keys sharing their first 12 bytes (one long probe chain), and
    compositions just below and just above the 40 % repeat threshold"""
    sm = engine.small_max()
    n = sm + 4096
    cap = 1
    while cap < 2 * n:
        cap <<= 1
    signer = _colliding_signers(cap - 1)
    (even_sk, even), (odd_sk, odd) = signer[0], signer[1]
    flip = lambda k: bytes([k[0] ^ 1]) + k[1:]
    ue = [_update(even_sk, j) for j in range(32)]
    uo = [_update(odd_sk, j) for j in range(32)]
    rng = np.random.default_rng(8600)
    # 02||x and 03||x of the same x, both ways round
    msgs, signers, want = [], [], []
    for i in range(n):
        c = int(rng.integers(4))
        u = (ue if c < 2 else uo)[i % 32]
        k = (even, flip(even), odd, flip(odd))[c]
        msgs.append(u), signers.append(k), want.append(c % 2)
    _gossip_both(engine, msgs, signers, np.array(want), 4, True)
    # one undecodable key (x >= p) repeated across hundreds of messages, interleaved with valid ones
    bad = b"\x02" + b"\xff" * 32
    sel = rng.random(n) < 0.1
    signers2 = [bad if s else k for s, k in zip(sel, signers)]
    want2 = np.where(sel, 1, want)
    assert sel.sum() > 500
    _gossip_both(engine, msgs, signers2, want2, 5, True)
    # 256 made-up keys with the same first 12 bytes: one probe chain; they cannot be signed for
    made = [b"\x02" + b"\x5a" * 11 + hashlib.sha256(b"made/%d" % j).digest()[:21] for j in range(256)]
    sel = rng.random(n) < 0.3
    signers3 = [made[int(rng.integers(256))] if s else k for s, k in zip(sel, signers)]
    want3 = np.where(sel, 1, want)
    _gossip_both(engine, msgs, signers3, want3, 4 + len(set(signers3) - {even, odd, flip(even), flip(odd)}), True)
    # distinct keys at the threshold: distinct * 10 <= 6 n takes the shared tables, one more does not
    limit = n * 6 // 10
    for distinct, uses in ((limit, True), (limit + 1, False)):
        many = [b"\x03" + hashlib.sha256(b"many/%d" % j).digest() for j in range(distinct - 2)]
        signers4 = [even, odd] + many
        signers4 += [(even, odd)[i % 2] for i in range(n - len(signers4))]
        order = rng.permutation(n)
        signers4 = [signers4[i] for i in order]
        msgs4 = [ue[i % 32] if k == even else uo[i % 32] for i, k in enumerate(signers4)]
        want4 = np.array([0 if k in (even, odd) else 1 for k in signers4])
        _gossip_both(engine, msgs4, signers4, want4, distinct, uses)
