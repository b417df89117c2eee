"""CPU: no item changes another item's verdict, on the host build of the kernel headers (tests/host_emul).

The special items of tests/isolation.py (one per label of the constructed fixture, all the others) in 32 blocks of 32
items, block b holding the special at offset b: every offset of the prep kernel's 32-signature inversion and of the final
kernels' 16-item inversions, among a valid background and one with about 25 % flipped messages.  Flows: the throughput
data flow (emul_verify_batch) with and without the square root, the small-batch lane pairs, the shared-key path and
BIP-340 batch verification.  Ragged tails, two specials of different classes in one 16-item unit, whole units of one
special and a seeded permutation as well.  The host build runs items one after another, so this catches arithmetic
faults in the batched products, not warp divergence: tests/test_gpu_isolation.py runs the same catalogue on the device."""
import ctypes
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from tests import isolation as I
from tests.util import P as ptr

BLOCKS = SIZE = 32
N_ITEMS = BLOCKS * SIZE
# (kind, exact): exact 1 = the plain flow with the square root, 0 = the flows without it (kinds 0 and 2)
FLOWS = ((0, 1), (0, 0), (1, 1), (2, 1), (2, 0))


def subset(kind):
    """the catalogue with one item per label of the constructed fixture"""
    seen, out = set(), []
    for sp in I.catalogue(kind):
        base = sp.label.split("#")[0]
        if sp.label.startswith("group.") and base in seen:
            continue
        seen.add(base)
        out.append(sp)
    return out


@pytest.fixture(scope="module")
def host(emul):
    emul.emul_gtable_build()
    emul.emul_last_exact_count.restype = ctypes.c_size_t
    yield emul
    emul.emul_set_ecdsa33_exact(0)


def backgrounds(kind, n=N_ITEMS):
    bg = I.host_background(kind, n)
    return {"valid": bg, "flipped": I.with_flips(bg, 900 + kind)}


def run(fn, kind, msg, key, sig):
    out = np.zeros(msg.shape[0], np.uint8)
    fn(kind, ptr(msg), ptr(key), ptr(sig), ctypes.c_size_t(msg.shape[0]), ptr(out))
    return out


def pool_map(f, jobs):
    """the host build's verifiers release the interpreter lock: one job per CPU"""
    with ThreadPoolExecutor(os.cpu_count() or 1) as ex:
        return list(ex.map(f, jobs))


def test_special_classes_match_the_host_build(host):
    """every special's own verdict; the 'exact' specials are handed to the plain path by the flows without the square
    root (emul_last_exact_count), the 'parse' ones are not (they are rejected before the curve work)"""
    try:
        host.emul_set_ecdsa33_exact(0)
        for kind in (0, 2):
            for sp in I.catalogue(kind):
                got = run(host.emul_verify_batch, kind, sp.msg[None], sp.key[None], sp.sig[None])
                assert got[0] == sp.want, sp
                if sp.cls in ("exact", "parse"):
                    assert (host.emul_last_exact_count() == 1) == (sp.cls == "exact"), sp
        host.emul_set_ecdsa33_exact(1)
        for kind in (0, 1, 2):
            for sp in I.catalogue(kind):
                assert run(host.emul_verify_batch, kind, sp.msg[None], sp.key[None], sp.sig[None])[0] == sp.want, sp
    finally:
        host.emul_set_ecdsa33_exact(0)


def test_block_layout_throughput_flows(host):
    """every special at every offset of a 32-item block, both backgrounds, every throughput flow: the whole verdict
    vector equals the expected one"""
    cov = I.Coverage()
    failures = []
    pos = I.block_positions(BLOCKS, SIZE)
    try:
        for kind, exact in FLOWS:
            host.emul_set_ecdsa33_exact(exact)
            bgs = backgrounds(kind)
            jobs = [(sp, name) for sp in subset(kind) for name in bgs]

            def one(job):
                sp, name = job
                msg, key, sig, want = I.block_layout(bgs[name], sp, BLOCKS, SIZE)
                return sp, name, run(host.emul_verify_batch, kind, msg, key, sig), want

            for sp, name, got, want in pool_map(one, jobs):
                bad = I.mismatch(got, want, {int(p): sp for p in pos}, SIZE)
                if bad:
                    failures.append(f"kind {kind} exact {exact} background {name}: {sp.label}\n{bad}")
                cov.add(f"batch.exact{exact}", sp, pos, SIZE)
    finally:
        host.emul_set_ecdsa33_exact(0)
    assert not failures, "\n".join(failures[:8])
    routes = {0: ["batch.exact1", "batch.exact0"], 1: ["batch.exact1"], 2: ["batch.exact1", "batch.exact0"]}
    assert not cov.missing(routes, {k: subset(k) for k in routes}, range(SIZE))
    # the final stages saw specials handed to the plain path and specials rejected before them beside pending items
    for kind in (0, 2):
        assert {sp.cls for sp in subset(kind)} >= {"exact", "parse"}, kind


def test_tails_pairs_full_units_and_permutation(host):
    """the special as the last item of n = 1024 + r (r = 1, 15, 17, 31); two specials of different classes in each
    16-item unit; 32-item units made of one special; and the pair batch shuffled: verdicts follow the items"""
    failures = []
    try:
        for kind, exact in FLOWS:
            host.emul_set_ecdsa33_exact(exact)
            specials = subset(kind)
            bg = backgrounds(kind, N_ITEMS + 31)["flipped"]
            one_per_class = list({sp.cls: sp for sp in specials}.values())
            jobs = [(r, sp) for r in (1, 15, 17, 31) for sp in one_per_class]

            def tail(job):
                r, sp = job
                n = N_ITEMS + r
                msg, key, sig, want = I.place(bg, n, {n - 1: sp})
                return r, sp, run(host.emul_verify_batch, kind, msg, key, sig), want

            for r, sp, got, want in pool_map(tail, jobs):
                bad = I.mismatch(got, want, {N_ITEMS + r - 1: sp}, 16)
                if bad:
                    failures.append(f"kind {kind} exact {exact} tail r = {r}: {sp.label}\n{bad}")
            layouts = [("pairs", N_ITEMS, I.pair_layout(specials, N_ITEMS, 40 + kind)), ("full units",) + I.full_unit_layout(specials)]
            for name, n, placed in layouts:
                big = backgrounds(kind, n)["flipped"]
                msg, key, sig, want = I.place(big, n, placed)
                got = run(host.emul_verify_batch, kind, msg, key, sig)
                bad = I.mismatch(got, want, placed, 32)
                if bad:
                    failures.append(f"kind {kind} exact {exact} {name}\n{bad}")
                perm = np.random.default_rng(50 + kind).permutation(n)
                got2 = run(host.emul_verify_batch, kind, msg[perm], key[perm], sig[perm])
                assert np.array_equal(got2, got[perm]), (kind, exact, name, "permuted")
    finally:
        host.emul_set_ecdsa33_exact(0)
    assert not failures, "\n".join(failures[:8])


def test_small_batch_pairs(host):
    """the small-batch path with its half ladders on lane pairs: each special at offsets 0 and 33 of 64 items"""
    failures = []
    placed_at = (0, 33)
    try:
        for kind, exact in ((0, 1), (1, 1), (2, 1), (2, 0)):
            host.emul_set_ecdsa33_exact(exact)
            bg = backgrounds(kind, 64)["flipped"]

            def one(sp):
                msg, key, sig, want = I.place(bg, 64, {p: sp for p in placed_at})
                return sp, run(host.emul_verify_small_pair_batch, kind, msg, key, sig), want

            for sp, got, want in pool_map(one, subset(kind)):
                bad = I.mismatch(got, want, {p: sp for p in placed_at}, 32)
                if bad:
                    failures.append(f"kind {kind} exact {exact}: {sp.label}\n{bad}")
    finally:
        host.emul_set_ecdsa33_exact(0)
    assert not failures, "\n".join(failures[:8])


def samekey_batch(sp, n, blocks, size, seed):
    """a shared-key batch for an ECDSA special: background signed with the special's own secret key (any key for a
    signature that does not parse), the special at offset b of block b.  A key that does not decode rejects everything."""
    d = sp.d if sp.d is not None else I.BASE_D
    bg = I.with_flips(I.samekey_background(sp.kind, d, n), seed)
    msg, _, sig, want = I.block_layout(bg, sp, blocks, size)
    if sp.label.startswith("key."):
        want[:] = 0
    return sp.key, msg, sig, want


def samekey_specials(kind, specials):
    """the specials whose key is known by its secret or does not decode"""
    return [sp for sp in specials if sp.d is not None or sp.label.startswith("key.")]


def test_shared_key_path(host):
    """the shared-key path (one table for the key, one inversion mod n per 32 signatures)"""
    failures = []
    pos = I.block_positions(BLOCKS, SIZE)
    for kind in (0, 1):
        def one(sp):
            key, msg, sig, want = samekey_batch(sp, N_ITEMS, BLOCKS, SIZE, 950 + kind)
            out = np.zeros(N_ITEMS, np.uint8)
            host.emul_verify_samekey(kind, ptr(key), ptr(msg), ptr(sig), ctypes.c_size_t(N_ITEMS), ptr(out))
            return sp, out, want

        specials = samekey_specials(kind, subset(kind))
        # only the reference's edge cases are left out: their keys come without a secret
        assert all(sp.label.startswith("edge.") for sp in subset(kind) if sp not in specials)
        for sp, got, want in pool_map(one, specials):
            bad = I.mismatch(got, want, {int(p): sp for p in pos}, SIZE)
            if bad:
                failures.append(f"kind {kind}: {sp.label}\n{bad}")
    assert not failures, "\n".join(failures[:8])


def test_bip340_batch_groups(host):
    """BIP-340 batch verification, 2 groups of 1024: the special at every offset of 32 blocks in group 0.  An item
    that fails the encoding check drops out (ok 0, both groups hold); a valid one leaves both groups holding; any other
    invalid one fails group 0 and only group 0."""
    seed = np.arange(32, dtype=np.uint8)
    n = 2048
    bg = I.host_background(2, n)
    pos = I.block_positions(BLOCKS, SIZE)

    def one(sp):
        msg, key, sig, want = I.place(bg, n, {int(p): sp for p in pos})
        ok = np.zeros(n, np.uint8)
        gok = np.zeros(2, np.uint8)
        host.emul_schnorr_batch(ptr(msg), ptr(key), ptr(sig), ctypes.c_size_t(n), ptr(seed), ptr(ok), ptr(gok))
        return sp, ok, gok

    specials = list(I.catalogue(2))
    for sp, ok, gok in pool_map(one, specials):
        want_ok = np.ones(n, np.uint8)
        want_ok[pos] = sp.sb_encoding
        assert np.array_equal(ok, want_ok), (sp.label, np.nonzero(ok != want_ok)[0][:8])
        holds = sp.want == 1 or not sp.sb_encoding
        assert list(gok) == [int(holds), 1], (sp.label, list(gok))
    assert any(sp.want for sp in specials) and any(not sp.sb_encoding for sp in specials)
