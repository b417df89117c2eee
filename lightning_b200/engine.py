"""ctypes binding of libcln_sigverify.so — the Python mirror of include/cln_sigverify.h.

The method names follow the reference surface they stand in for (bitcoin/signature.h:
check_signed_hash :85, check_schnorr_sig :129; common/node_id.h: check_signed_hash_nodeid :80;
bitcoin/shadouble.h: sha256_double), batched.  There is no Python or CPU implementation behind
this class: if the CUDA library or a GPU is missing, construction raises.
"""
import ctypes
import errno
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("SV_LIB") or os.path.join(_HERE, "libcln_sigverify.so")  # SV_LIB: another build of the library (dev)

SV_ERR_ARG, SV_ERR_IO = -4, -5  # sv_status values a caller of sv_prune/repair_gossip_store_fd tells apart
KIND_ECDSA33 = 0
KIND_ECDSA_XY = 1
KIND_SCHNORR = 2
KEY_SIZE = {KIND_ECDSA33: 33, KIND_ECDSA_XY: 64, KIND_SCHNORR: 32}
STG_IN_WORDS, STG_OUT_WORDS = 64, 200  # SV_STG_IN_WORDS / SV_STG_OUT_WORDS: record widths of the group self test

_c8 = ctypes.POINTER(ctypes.c_uint8)


class EngineError(RuntimeError):
    pass


class SvTx(ctypes.Structure):
    """sv_tx (include/cln_sigverify.h): the BIP143-relevant fields of a one-input one-output segwit transaction."""
    _fields_ = [("version", ctypes.c_uint32), ("locktime", ctypes.c_uint32), ("sequence", ctypes.c_uint32),
                ("sighash_type", ctypes.c_uint32), ("prev_txid", ctypes.c_uint8 * 32), ("prev_index", ctypes.c_uint32),
                ("script_off", ctypes.c_uint32), ("script_len", ctypes.c_uint32), ("out_script_off", ctypes.c_uint32),
                ("out_script_len", ctypes.c_uint32), ("flags", ctypes.c_uint32), ("input_amount", ctypes.c_uint64),
                ("output_amount", ctypes.c_uint64), ("prevouts_off", ctypes.c_uint32), ("prevouts_len", ctypes.c_uint32),
                ("sequences_off", ctypes.c_uint32), ("sequences_len", ctypes.c_uint32)]


class SvGossipStoreSummary(ctypes.Structure):
    """sv_gossip_store_summary (include/cln_sigverify.h)"""
    _fields_ = [("version", ctypes.c_uint32), ("stop", ctypes.c_int32)] + [(f, ctypes.c_uint64) for f in (
        "end_offset", "ended_equivalent_offset", "records", "good", "bad_signature", "malformed", "no_channel", "wrong_chain",
        "bad_order", "deleted", "store_records", "unknown", "not_reached", "redundant_announcements",
        "updates_without_channel")]


# record statuses of verify_gossip_store besides the signature statuses (include/cln_sigverify.h SV_GS_*)
GS_EOF, GS_DELETED, GS_STORE_RECORD, GS_UNKNOWN, GS_NOT_REACHED = 0, 16, 17, 18, 19
GS_INCOMPLETE, GS_PARTIAL, GS_TRUNCATED, GS_BAD_CRC, GS_ENDED, GS_NO_AMOUNT = 32, 33, 34, 35, 36, 37
GS_NO_HOLDER = (1 << 64) - 1


class SvGossipPruneSummary(ctypes.Structure):
    """sv_gossip_prune_summary (include/cln_sigverify.h)"""
    _fields_ = [("version", ctypes.c_uint32), ("stop", ctypes.c_int32)] + [(f, ctypes.c_uint64) for f in (
        "end_offset", "records", "pruned", "bad_crc", "truncated", "message", "redundant", "no_channel", "signature",
        "amount", "unknown", "reverified")]


# why prune_gossip_store deletes a record (include/cln_sigverify.h SV_GP_*; 0 = kept)
GP_KEPT, GP_BAD_CRC, GP_TRUNCATED, GP_MESSAGE, GP_REDUNDANT, GP_NO_CHANNEL, GP_SIGNATURE, GP_AMOUNT, GP_UNKNOWN = range(9)
GP_REASONS = ("kept", "bad_crc", "truncated", "message", "redundant", "no_channel", "signature", "amount", "unknown")


class SvFundingTable(ctypes.Structure):
    """sv_funding_table (include/cln_sigverify.h)"""
    _fields_ = [("scid", ctypes.c_void_p), ("satoshis", ctypes.c_void_p), ("script34", ctypes.c_void_p),
                ("n_outputs", ctypes.c_size_t), ("blocks", ctypes.c_void_p), ("n_blocks", ctypes.c_size_t)]


class SvGossipFundingSummary(ctypes.Structure):
    """sv_gossip_funding_summary (include/cln_sigverify.h)"""
    _fields_ = [(f, ctypes.c_uint64) for f in ("checked", "funded", "unchecked", "no_txout", "script", "amount", "dying",
                                               "deleted")]


# the funding verdict of a channel_announcement (include/cln_sigverify.h SV_GF_*; 0 = none); GP_FUNDING: the prune's
# reason for deleting an announcement whose verdict is NO_TXOUT, SCRIPT or AMOUNT
GF_NONE, GF_FUNDED, GF_UNCHECKED, GF_DYING, GF_NO_TXOUT, GF_SCRIPT, GF_AMOUNT = range(7)
GP_FUNDING = 9


def _funding_table(funding):
    """the sv_funding_table of a lightning_b200.funding.FundingTable (its arrays stay referenced by the table)"""
    t = SvFundingTable(funding.scid.ctypes.data, funding.satoshis.ctypes.data, funding.script.ctypes.data, len(funding),
                       funding.blocks.ctypes.data, funding.blocks.size)
    t._keep = funding
    return t


class SvInfo(ctypes.Structure):
    _fields_ = [("device", ctypes.c_int), ("sm_count", ctypes.c_int), ("main_block", ctypes.c_int),
                ("main_grid", ctypes.c_int), ("main_regs", ctypes.c_int), ("gtable_bytes", ctypes.c_size_t),
                ("scratch_bytes", ctypes.c_size_t), ("launches", ctypes.c_ulonglong), ("l2_persist_bytes", ctypes.c_size_t), ("l2_max_persist_bytes", ctypes.c_size_t)]


def load_library():
    if not os.path.exists(LIB_PATH):
        raise EngineError(
            f"{LIB_PATH} is missing: build it with `python -m lightning_b200.build` "
            "(nvcc, sm_90a). There is no CPU fallback.")
    lib = ctypes.CDLL(LIB_PATH, use_errno=True)  # errno: sv_prune_gossip_store_fd says why a file was refused
    vp, sz, i = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int
    lib.sv_create.argtypes = [ctypes.POINTER(vp), i]
    lib.sv_destroy.argtypes = [vp]
    lib.sv_destroy.restype = None
    lib.sv_last_error.argtypes = [vp]
    lib.sv_last_error.restype = ctypes.c_char_p
    lib.sv_key_size.argtypes = [i]
    lib.sv_key_size.restype = sz
    lib.sv_verify_host.argtypes = [vp, i, vp, vp, vp, sz, vp]
    lib.sv_verify_host_raw.argtypes = [vp, i, vp, sz, vp, vp, vp, vp, sz, vp]
    lib.sv_verify_device.argtypes = [vp, i, vp, vp, vp, sz, vp, vp, vp]
    lib.sv_verify_gossip_host.argtypes = [vp, vp, sz, vp, vp, sz, vp, vp]
    lib.sv_verify_gossip_burst_host.argtypes = [vp, vp, vp, sz, vp, vp, sz, vp, vp, vp]
    lib.sv_last_gossip_repairs.argtypes = [vp]
    lib.sv_last_gossip_repairs.restype = ctypes.c_uint
    lib.sv_gossip_store_count.argtypes = [vp, sz]
    lib.sv_gossip_store_count.restype = sz
    lib.sv_verify_gossip_store_host.argtypes = [vp, vp, sz, vp, vp, vp, vp, vp, sz, ctypes.POINTER(SvGossipStoreSummary)]
    lib.sv_get_last_gossip_store_timing.argtypes = [vp, ctypes.POINTER(ctypes.c_float)]
    lib.sv_gossip_prune_count.argtypes = [vp, sz]
    lib.sv_gossip_prune_count.restype = sz
    lib.sv_prune_gossip_store_host.argtypes = [vp, vp, sz, vp, vp, vp, vp, vp, vp, sz, ctypes.POINTER(SvGossipPruneSummary)]
    lib.sv_get_last_gossip_prune_timing.argtypes = [vp, ctypes.POINTER(ctypes.c_float)]
    lib.sv_verify_gossip_store_funding_host.argtypes = [vp, vp, sz, vp, ctypes.POINTER(SvFundingTable), vp, vp, vp, vp, vp,
                                                        sz, ctypes.POINTER(SvGossipStoreSummary),
                                                        ctypes.POINTER(SvGossipFundingSummary)]
    lib.sv_prune_gossip_store_funding_host.argtypes = [vp, vp, sz, vp, ctypes.POINTER(SvFundingTable), vp, vp, vp, vp, vp,
                                                       vp, sz, ctypes.POINTER(SvGossipPruneSummary),
                                                       ctypes.POINTER(SvGossipFundingSummary)]
    lib.sv_get_last_gossip_funding_timing.argtypes = [vp, ctypes.POINTER(ctypes.c_float)]
    lib.sv_prune_gossip_store_fd.argtypes = [vp, i, ctypes.c_uint64, vp, ctypes.POINTER(SvGossipPruneSummary)]
    lib.sv_repair_gossip_store_fd.argtypes = [vp, i, ctypes.c_uint64, vp, ctypes.POINTER(SvGossipPruneSummary),
                                              ctypes.POINTER(ctypes.c_uint64)]
    lib.sv_gossip_prune_cut.restype = ctypes.c_uint64
    lib.sv_gossip_prune_cut.argtypes = [ctypes.POINTER(SvGossipPruneSummary), ctypes.c_char_p, ctypes.c_uint64]
    lib.sv_verify_tx_host.argtypes = [vp, i, vp, vp, sz, vp, vp, sz, vp, vp]
    lib.sv_grind_tx_fee_host.argtypes = [vp, i, vp, vp, sz, vp, vp, ctypes.c_uint64, ctypes.c_uint32, ctypes.c_uint32,
                                         ctypes.POINTER(ctypes.c_int64), ctypes.POINTER(ctypes.c_uint64)]
    lib.sv_verify_samekey_host.argtypes = [vp, i, vp, vp, vp, sz, vp]
    lib.sv_verify_bolt12_host.argtypes = [vp, ctypes.c_char_p, ctypes.c_char_p, vp, sz, vp, vp, vp, vp, sz, vp, vp]
    lib.sv_verify_bolt12_tagged_host.argtypes = [vp, sz, vp, vp, vp, vp, sz, vp, vp, vp, vp, sz, vp, vp]
    lib.sv_get_last_bolt12_timing.argtypes = [vp, ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_float)]
    lib.sv_sync.argtypes = [vp, vp]
    lib.sv_get_stream.argtypes = [vp]
    lib.sv_set_profiling.argtypes = [vp, i]
    lib.sv_get_last_timing.argtypes = [vp, ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_float)]
    lib.sv_get_stream.restype = vp
    lib.sv_enqueue.argtypes = [vp, i, vp, vp, vp]
    lib.sv_enqueue.restype = ctypes.c_long
    lib.sv_pending.argtypes = [vp]
    lib.sv_pending.restype = sz
    lib.sv_flush.argtypes = [vp, vp, sz]
    lib.sv_sha256d_host.argtypes = [vp, vp, sz, vp, vp, sz, vp]
    lib.sv_pubkey_parse_host.argtypes = [vp, vp, sz, vp, vp]
    lib.sv_synth_device.argtypes = [vp, i, ctypes.c_uint64, sz, vp, vp, vp, vp]
    lib.sv_selftest_host.argtypes = [vp, i, vp, vp, sz, vp]
    lib.sv_selftest_group_host.argtypes = [vp, i, vp, sz, vp]
    lib.sv_verify_mixed_host.argtypes = [vp, vp, vp, vp, vp, sz, vp]
    lib.sv_verify_mixed_device.argtypes = [vp, vp, vp, vp, vp, sz, vp, vp]
    lib.sv_verify_schnorr_batch_host.argtypes = [vp, vp, vp, vp, sz, vp, vp, vp, vp]
    lib.sv_set_dedup.argtypes = [vp, i]
    lib.sv_set_nosqrt.argtypes = [vp, i]
    lib.sv_last_distinct_keys.argtypes = [vp]
    lib.sv_last_distinct_keys.restype = ctypes.c_uint
    lib.sv_set_small_max.argtypes = [vp, sz]
    lib.sv_get_small_max.argtypes = [vp]
    lib.sv_get_small_max.restype = sz
    lib.sv_get_info.argtypes = [vp, ctypes.POINTER(SvInfo)]
    lib.sv_probe.argtypes = [vp, i, ctypes.POINTER(ctypes.c_double)]
    lib.sv_probe_imad_peak.argtypes = [vp, ctypes.POINTER(ctypes.c_double)]
    lib.sv_host_alloc.argtypes = [sz]
    lib.sv_host_alloc.restype = vp
    lib.sv_host_free.argtypes = [vp]
    lib.sv_host_free.restype = None
    return lib


def _u8(a, shape_tail):
    a = np.ascontiguousarray(a, dtype=np.uint8)
    if a.ndim == 1:
        a = a.reshape(-1, shape_tail)
    if a.shape[1] != shape_tail:
        raise ValueError(f"expected (*, {shape_tail}) uint8, got {a.shape}")
    return a


def _chain_hash(h):
    chain = np.frombuffer(bytes(h), dtype=np.uint8)
    if chain.size != 32:
        raise ValueError("chain_hash must be 32 bytes")
    return chain


class SigVerifier:
    """One engine context on one GPU (sv_ctx)."""

    def __init__(self, device=0):
        self.lib = load_library()
        self._ctx = ctypes.c_void_p()
        rc = self.lib.sv_create(ctypes.byref(self._ctx), int(device))
        if rc != 0:
            msg = self.lib.sv_last_error(None).decode()
            self._ctx = ctypes.c_void_p()
            raise EngineError(f"sv_create(device={device}) failed ({rc}): {msg}")
        self.device = int(device)

    def close(self):
        if getattr(self, "_ctx", None) and self._ctx.value:
            self.lib.sv_destroy(self._ctx)
            self._ctx = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc, what):
        if rc != 0:
            raise EngineError(f"{what} failed ({rc}): {self.lib.sv_last_error(self._ctx).decode()}")

    # ---- host-buffer API -------------------------------------------------------------------
    def verify(self, kind, msg32, key, sig64):
        """Batch verify; returns a uint8 verdict vector.  Host numpy arrays in, host array out."""
        msg32 = _u8(msg32, 32)
        key = _u8(key, KEY_SIZE[kind])
        sig64 = _u8(sig64, 64)
        n = msg32.shape[0]
        if key.shape[0] != n or sig64.shape[0] != n:
            raise ValueError("length mismatch")
        out = np.zeros(n, dtype=np.uint8)
        self._check(self.lib.sv_verify_host(self._ctx, kind, msg32.ctypes.data, key.ctypes.data, sig64.ctypes.data,
                                            n, out.ctypes.data), "sv_verify_host")
        return out

    def check_signed_hash(self, hash32, sig64, pubxy64):
        """bitcoin/signature.c:174 check_signed_hash, batched (pre-decompressed keys)."""
        return self.verify(KIND_ECDSA_XY, hash32, pubxy64, sig64)

    def check_signed_hash_nodeid(self, hash32, sig64, node_id33):
        """common/node_id.c:72 check_signed_hash_nodeid, batched (33-byte keys)."""
        return self.verify(KIND_ECDSA33, hash32, node_id33, sig64)

    def check_schnorr_sig(self, hash32, xonly32, sig64):
        """bitcoin/signature.c:408 check_schnorr_sig, batched (x-only keys)."""
        return self.verify(KIND_SCHNORR, hash32, xonly32, sig64)

    def verify_raw(self, kind, data, off, length, key, sig64):
        """Verify over SHA256d(data[off:off+len]) computed on the device (gossipd/sigcheck.c path)."""
        data = np.ascontiguousarray(data, dtype=np.uint8).reshape(-1)
        off = np.ascontiguousarray(off, dtype=np.uint64)
        length = np.ascontiguousarray(length, dtype=np.uint32)
        key = _u8(key, KEY_SIZE[kind])
        sig64 = _u8(sig64, 64)
        n = off.shape[0]
        out = np.zeros(n, dtype=np.uint8)
        self._check(self.lib.sv_verify_host_raw(self._ctx, kind, data.ctypes.data, data.size, off.ctypes.data,
                                                length.ctypes.data, key.ctypes.data, sig64.ctypes.data, n,
                                                out.ctypes.data), "sv_verify_host_raw")
        return out

    def verify_gossip(self, msgs, cu_signers=None):
        """Raw gossip wire messages in, one status per message out (0 ok, 1..4 first bad signature, -1 malformed);
        the device slices, hashes and verifies (gossipd/sigcheck.c, batched).  cu_signers: (n,33) or None."""
        lens = np.array([len(m) for m in msgs], dtype=np.uint32)
        offs = np.concatenate([[0], np.cumsum(lens[:-1], dtype=np.uint64)]).astype(np.uint64) if len(msgs) else np.zeros(0, np.uint64)
        blob = np.frombuffer(b"".join(bytes(m) for m in msgs), dtype=np.uint8)
        n = len(msgs)
        status = np.zeros(max(n, 1), dtype=np.int32)
        sg = None
        if cu_signers is not None:
            sg = _u8(cu_signers, 33)
        self._check(self.lib.sv_verify_gossip_host(self._ctx, blob.ctypes.data, blob.size, offs.ctypes.data, lens.ctypes.data, n,
                                                   sg.ctypes.data if sg is not None else None, status.ctypes.data),
                    "sv_verify_gossip_host")
        return status[:n]

    def verify_gossip_burst(self, msgs, chain_hash, signer_kind=None, signers=None):
        """A burst of raw gossip messages of any types; a channel_update's signer comes from the batch's own
        channel_announcements (signer_kind 0), from signers[m] (1), or from the batch with signers[m] as the source peer's
        fallback (2).  Returns int32 statuses: 0 ok, 1..4 first bad signature, 5 verified under the source peer, -1
        malformed, -2 no channel, -3 other chain, -4 node ids out of order (cln_sigverify.h)."""
        n = len(msgs)
        lens = np.array([len(m) for m in msgs], dtype=np.uint32)
        offs = np.concatenate([[0], np.cumsum(lens[:-1], dtype=np.uint64)]).astype(np.uint64) if n else np.zeros(0, np.uint64)
        blob = np.frombuffer(b"".join(bytes(m) for m in msgs), dtype=np.uint8)
        chain = _chain_hash(chain_hash)
        kinds = None if signer_kind is None else np.ascontiguousarray(signer_kind, dtype=np.uint8).reshape(-1)
        if kinds is not None and kinds.size != n:
            raise ValueError("signer_kind: one byte per message")
        sg = None if signers is None else _u8(signers, 33)
        if sg is not None and sg.shape[0] != n:
            raise ValueError("signers: one 33-byte key per message")
        status = np.zeros(max(n, 1), dtype=np.int32)
        self._check(self.lib.sv_verify_gossip_burst_host(
            self._ctx, chain.ctypes.data, blob.ctypes.data, blob.size, offs.ctypes.data, lens.ctypes.data, n,
            kinds.ctypes.data if kinds is not None else None, sg.ctypes.data if sg is not None else None,
            status.ctypes.data), "sv_verify_gossip_burst_host")
        return status[:n]

    def last_gossip_repairs(self):
        """updates the last gossip burst re-resolved in its repair round (their first candidate announcement failed)"""
        return int(self.lib.sv_last_gossip_repairs(self._ctx))

    def verify_gossip_store(self, store, chain_hash=None, capacity=None, funding=None):
        """A whole gossip_store (bytes, version byte included), walked as gossmap's map_catchup walks it, every record
        checksum and every signature checked on the device.  Returns (rec_off uint64, rec_type uint16, rec_status int32,
        rec_holder uint64, summary dict): one entry per record the walk reads; rec_status is a signature status for
        256/257/258 (0, 1..4, -1, -2 no channel, and with chain_hash -3 / -4) or a GS_* record status; rec_holder is the
        header offset of the announcement holding the channel (updates, redundant announcements), else GS_NO_HOLDER.
        capacity: entries to provide (default: sv_gossip_store_count).
        funding: a lightning_b200.funding.FundingTable, or None.  With a table every announcement is also checked against
        lightningd's funding outputs (sv_verify_gossip_store_funding_host), and the call returns two more items:
        rec_funding uint8 (GF_* verdict per record) and the funding summary dict."""
        buf = np.frombuffer(bytes(store), dtype=np.uint8)
        chain = None if chain_hash is None else _chain_hash(chain_hash)
        n = int(self.lib.sv_gossip_store_count(buf.ctypes.data, buf.size)) if capacity is None else int(capacity)
        off = np.zeros(max(n, 1), np.uint64)
        typ = np.zeros(max(n, 1), np.uint16)
        status = np.zeros(max(n, 1), np.int32)
        holder = np.zeros(max(n, 1), np.uint64)
        s = SvGossipStoreSummary()
        if funding is None:
            self._check(self.lib.sv_verify_gossip_store_host(
                self._ctx, buf.ctypes.data, buf.size, chain.ctypes.data if chain is not None else None, off.ctypes.data,
                typ.ctypes.data, status.ctypes.data, holder.ctypes.data, n, ctypes.byref(s)), "sv_verify_gossip_store_host")
        else:
            fund, fs, table = np.zeros(max(n, 1), np.uint8), SvGossipFundingSummary(), _funding_table(funding)
            self._check(self.lib.sv_verify_gossip_store_funding_host(
                self._ctx, buf.ctypes.data, buf.size, chain.ctypes.data if chain is not None else None, ctypes.byref(table),
                off.ctypes.data, typ.ctypes.data, status.ctypes.data, holder.ctypes.data, fund.ctypes.data, n,
                ctypes.byref(s), ctypes.byref(fs)), "sv_verify_gossip_store_funding_host")
        summary = {f: getattr(s, f) for f, _ in SvGossipStoreSummary._fields_}
        k = s.records
        if funding is None:
            return off[:k], typ[:k], status[:k], holder[:k], summary
        return off[:k], typ[:k], status[:k], holder[:k], summary, fund[:k], {f: getattr(fs, f) for f, _ in fs._fields_}

    def last_gossip_store_timing(self):
        """(header walk, H2D, checksums, verification) in ms of the last verify_gossip_store (profiling mode)"""
        ms = (ctypes.c_float * 4)()
        self._check(self.lib.sv_get_last_gossip_store_timing(self._ctx, ms), "sv_get_last_gossip_store_timing")
        return tuple(ms)

    def prune_gossip_store(self, store, chain_hash=None, capacity=None, funding=None):
        """Mark every record of a gossip_store that gossmap should not trust as deleted (flag bit 0x8000), so that
        gossipd's strict load accepts the store and keeps the rest.  Returns (pruned_bytes, records, summary): the store
        with those bits set (same length; the input is not changed), records = (rec_off uint64, rec_type uint16,
        rec_status int32 (the first-round status), rec_pruned uint8 (GP_* reason, 0 = kept)), and the summary dict with
        the deletions per reason.  capacity: entries to provide (default: sv_gossip_prune_count).
        funding: a lightning_b200.funding.FundingTable, or None.  With a table the announcements gossipd would have
        refused for their funding output are deleted too (GP_FUNDING, sv_prune_gossip_store_funding_host; summary
        "pruned" counts them), and the call returns two more items: rec_funding uint8 (GF_* verdict per record) and
        the funding summary dict ("deleted": the funding deletions)."""
        buf = np.frombuffer(bytes(store), dtype=np.uint8)
        chain = None if chain_hash is None else _chain_hash(chain_hash)
        n = int(self.lib.sv_gossip_prune_count(buf.ctypes.data, buf.size)) if capacity is None else int(capacity)
        out = np.empty(max(buf.size, 1), np.uint8)
        off = np.zeros(max(n, 1), np.uint64)
        typ = np.zeros(max(n, 1), np.uint16)
        status = np.zeros(max(n, 1), np.int32)
        pruned = np.zeros(max(n, 1), np.uint8)
        s = SvGossipPruneSummary()
        if funding is None:
            self._check(self.lib.sv_prune_gossip_store_host(
                self._ctx, buf.ctypes.data, buf.size, chain.ctypes.data if chain is not None else None, out.ctypes.data,
                off.ctypes.data, typ.ctypes.data, status.ctypes.data, pruned.ctypes.data, n, ctypes.byref(s)),
                "sv_prune_gossip_store_host")
        else:
            fund, fs, table = np.zeros(max(n, 1), np.uint8), SvGossipFundingSummary(), _funding_table(funding)
            self._check(self.lib.sv_prune_gossip_store_funding_host(
                self._ctx, buf.ctypes.data, buf.size, chain.ctypes.data if chain is not None else None, ctypes.byref(table),
                out.ctypes.data, off.ctypes.data, typ.ctypes.data, status.ctypes.data, pruned.ctypes.data, fund.ctypes.data,
                n, ctypes.byref(s), ctypes.byref(fs)), "sv_prune_gossip_store_funding_host")
        summary = {f: getattr(s, f) for f, _ in SvGossipPruneSummary._fields_}
        k = s.records
        if funding is None:
            return out[:buf.size].tobytes(), (off[:k], typ[:k], status[:k], pruned[:k]), summary
        return (out[:buf.size].tobytes(), (off[:k], typ[:k], status[:k], pruned[:k]), summary, fund[:k],
                {f: getattr(fs, f) for f, _ in fs._fields_})

    def prune_gossip_store_fd(self, fd, length, chain_hash=None):
        """prune_gossip_store on a FILE, in place (sv_prune_gossip_store_fd): the store is bytes [0, length) of fd, a
        regular file open for reading and writing; the flags of the records deleted are written back into it and the file
        is synced, no other byte changes.  Returns the summary dict prune_gossip_store returns.  A file the call cannot use
        or a store it refuses raises OSError with the call's errno (EINVAL, EBADF, or that of a failed read, write or
        fsync); an engine failure raises EngineError."""
        return self._store_fd(False, fd, length, chain_hash)[0]

    def repair_gossip_store_fd(self, fd, length, chain_hash=None):
        """prune_gossip_store_fd, then the file cut where a torn append begins (sv_repair_gossip_store_fd: an incomplete
        or partial last record, an announcement without its amount record, or a torn header; see gossip_prune_cut).
        Returns (the summary dict, new_len: where the file ends now).  Errors as prune_gossip_store_fd, and a failed
        ftruncate raises OSError too."""
        return self._store_fd(True, fd, length, chain_hash)

    def gossip_prune_cut(self, summary, pruned):
        """sv_gossip_prune_cut: where sv_repair_gossip_store_fd ends a store whose prune gave `summary` (a dict as
        prune_gossip_store returns) and the bytes `pruned`"""
        s = SvGossipPruneSummary(**{f: summary[f] for f, _ in SvGossipPruneSummary._fields_})
        pruned = bytes(pruned)
        return int(self.lib.sv_gossip_prune_cut(ctypes.byref(s), pruned, len(pruned)))

    def _store_fd(self, repair, fd, length, chain_hash):
        chain = None if chain_hash is None else _chain_hash(chain_hash)
        s, new_len = SvGossipPruneSummary(), ctypes.c_uint64(0)
        cp = chain.ctypes.data if chain is not None else None
        if repair:
            name = "sv_repair_gossip_store_fd"
            rc = self.lib.sv_repair_gossip_store_fd(self._ctx, int(fd), int(length), cp, ctypes.byref(s), ctypes.byref(new_len))
        else:
            name = "sv_prune_gossip_store_fd"
            rc = self.lib.sv_prune_gossip_store_fd(self._ctx, int(fd), int(length), cp, ctypes.byref(s))
        if rc in (SV_ERR_ARG, SV_ERR_IO):
            e = ctypes.get_errno() or errno.EINVAL
            raise OSError(e, f"{name}: {os.strerror(e)}")
        self._check(rc, name)
        return {f: getattr(s, f) for f, _ in SvGossipPruneSummary._fields_}, int(new_len.value)

    def last_gossip_prune_timing(self):
        """(header walk, first round, second round, flag write) in ms of the last prune_gossip_store (profiling mode)"""
        ms = (ctypes.c_float * 4)()
        self._check(self.lib.sv_get_last_gossip_prune_timing(self._ctx, ms), "sv_get_last_gossip_prune_timing")
        return tuple(ms)

    def last_gossip_funding_timing(self):
        """(table staging and sort, k_store_funding) in ms of the last funding call (profiling mode)"""
        ms = (ctypes.c_float * 2)()
        self._check(self.lib.sv_get_last_gossip_funding_timing(self._ctx, ms), "sv_get_last_gossip_funding_timing")
        return tuple(ms)

    def verify_samekey(self, kind, key, msg32, sig64):
        """n ECDSA signatures by ONE key (channeld's HTLC loop): the key's table is built once on the device."""
        msg32 = _u8(msg32, 32)
        sig64 = _u8(sig64, 64)
        k = np.ascontiguousarray(key, dtype=np.uint8).reshape(-1)
        assert k.size == KEY_SIZE[kind]
        n = msg32.shape[0]
        out = np.zeros(max(n, 1), dtype=np.uint8)
        self._check(self.lib.sv_verify_samekey_host(self._ctx, kind, k.ctypes.data, msg32.ctypes.data, sig64.ctypes.data, n,
                                                    out.ctypes.data), "sv_verify_samekey_host")
        return out[:n]

    def check_tx_sigs(self, kind, txs, scripts, key, sig64, want_sighash=False):
        """check_tx_sig (bitcoin/signature.c:194) for n one-input one-output transactions with the BIP143 sighash
        computed on the device.  txs: ctypes array of SvTx; scripts: bytes blob; key (n, keysize); sig64 (n, 64)."""
        n = len(txs)
        key = _u8(key, KEY_SIZE[kind])
        sig64 = _u8(sig64, 64)
        blob = np.frombuffer(bytes(scripts) if len(scripts) else b"\0", dtype=np.uint8)
        out = np.zeros(max(n, 1), dtype=np.uint8)
        sh = np.zeros((max(n, 1), 32), dtype=np.uint8)
        self._check(self.lib.sv_verify_tx_host(self._ctx, kind, ctypes.addressof(txs), blob.ctypes.data, len(scripts),
                                               key.ctypes.data, sig64.ctypes.data, n, out.ctypes.data,
                                               sh.ctypes.data if want_sighash else None), "sv_verify_tx_host")
        return (out[:n], sh[:n]) if want_sighash else out[:n]

    def grind_tx_fee(self, kind, tx, scripts, key, sig64, weight, min_feerate, max_feerate):
        """onchaind's HTLC fee grind (onchaind/onchaind.c:389-437) in one call: the first feerate in [min_feerate,
        max_feerate] whose fee = feerate * weight // 1000 makes sig64 verify for tx (an SvTx, flags 0) with its output set
        to input_amount - fee.  Returns (feerate, fee), or (None, 0) when none verifies."""
        k = np.ascontiguousarray(np.frombuffer(bytes(key), dtype=np.uint8))
        s = np.ascontiguousarray(np.frombuffer(bytes(sig64), dtype=np.uint8))
        if k.size != KEY_SIZE[kind] or s.size != 64:
            raise ValueError("key or signature of the wrong size")
        blob = np.frombuffer(bytes(scripts) if len(scripts) else b"\0", dtype=np.uint8)
        f, fee = ctypes.c_int64(), ctypes.c_uint64()
        self._check(self.lib.sv_grind_tx_fee_host(self._ctx, kind, ctypes.byref(tx), blob.ctypes.data, len(scripts),
                                                  k.ctypes.data, s.ctypes.data, int(weight), int(min_feerate),
                                                  int(max_feerate), ctypes.byref(f), ctypes.byref(fee)),
                    "sv_grind_tx_fee_host")
        return (None, 0) if f.value < 0 else (f.value, fee.value)

    def verify_bolt12(self, messagename, fieldname, streams, xonly, sig, want_sighash=False):
        """bolt12_check_signature (common/bolt12.c:80) for n raw TLV streams, Merkle root and sighash computed on the
        device.  streams: sequence of bytes-like; xonly (n, 32); sig (n, 64).  Returns int32 statuses (1 valid, 0 invalid,
        -1 not a TLV stream CLN parses, or empty), and with want_sighash also the (n, 32) sighashes (zeros where -1)."""
        lens = np.array([len(s) for s in streams], dtype=np.uint32)
        offs = np.zeros(len(streams), dtype=np.uint64)
        if len(streams) > 1:
            offs[1:] = np.cumsum(lens[:-1], dtype=np.uint64)
        blob = np.frombuffer(b"".join(bytes(s) for s in streams), dtype=np.uint8)
        return self.verify_bolt12_spans(messagename, fieldname, blob, offs, lens, xonly, sig, want_sighash)

    def verify_bolt12_spans(self, messagename, fieldname, blob, off, length, xonly, sig, want_sighash=False):
        """verify_bolt12 with the streams already laid out: stream i = blob[off[i]:off[i]+length[i]]."""
        blob = np.ascontiguousarray(blob, dtype=np.uint8).reshape(-1)
        off = np.ascontiguousarray(off, dtype=np.uint64)
        length = np.ascontiguousarray(length, dtype=np.uint32)
        xonly, sig = _u8(xonly, 32), _u8(sig, 64)
        n = off.shape[0]
        if length.shape[0] != n or xonly.shape[0] != n or sig.shape[0] != n:
            raise ValueError("length mismatch")
        status =np.zeros(max(n, 1), dtype=np.int32)
        sh = np.zeros((max(n, 1), 32), dtype=np.uint8)
        mn = messagename.encode() if isinstance(messagename, str) else bytes(messagename)
        fn = fieldname.encode() if isinstance(fieldname, str) else bytes(fieldname)
        self._check(self.lib.sv_verify_bolt12_host(self._ctx, mn, fn, blob.ctypes.data, blob.size, off.ctypes.data,
                                                   length.ctypes.data, xonly.ctypes.data, sig.ctypes.data, n,
                                                   status.ctypes.data, sh.ctypes.data if want_sighash else None),
                    "sv_verify_bolt12_host")
        return (status[:n], sh[:n]) if want_sighash else status[:n]

    def verify_bolt12_tagged(self, tags, tag_of, blob, off, length, xonly, sig, want_sighash=False):
        """verify_bolt12_spans with a tag per stream, in one pass: tags is a sequence of (messagename, fieldname) pairs,
        stream i is hashed under tags[tag_of[i]]."""
        blob = np.ascontiguousarray(blob, dtype=np.uint8).reshape(-1)
        off = np.ascontiguousarray(off, dtype=np.uint64)
        length = np.ascontiguousarray(length, dtype=np.uint32)
        tag_of = np.ascontiguousarray(tag_of, dtype=np.uint32)
        xonly, sig = _u8(xonly, 32), _u8(sig, 64)
        n = off.shape[0]
        if length.shape[0] != n or tag_of.shape[0] != n or xonly.shape[0] != n or sig.shape[0] != n:
            raise ValueError("length mismatch")
        enc = [(s.encode() if isinstance(s, str) else bytes(s)) for pair in tags for s in pair]  # alive through the call
        mn = (ctypes.c_char_p * max(len(tags), 1))(*enc[0::2])
        fn = (ctypes.c_char_p * max(len(tags), 1))(*enc[1::2])
        status = np.zeros(max(n, 1), dtype=np.int32)
        sh = np.zeros((max(n, 1), 32), dtype=np.uint8)
        self._check(self.lib.sv_verify_bolt12_tagged_host(self._ctx, len(tags), mn, fn, tag_of.ctypes.data, blob.ctypes.data,
                                                          blob.size, off.ctypes.data, length.ctypes.data, xonly.ctypes.data,
                                                          sig.ctypes.data, n, status.ctypes.data,
                                                          sh.ctypes.data if want_sighash else None),
                    "sv_verify_bolt12_tagged_host")
        return (status[:n], sh[:n]) if want_sighash else status[:n]

    def last_bolt12_timing(self):
        """(merkle_ms, verify_ms) device time of the last verify_bolt12 call; needs set_profiling(True)."""
        a, b = ctypes.c_float(), ctypes.c_float()
        self._check(self.lib.sv_get_last_bolt12_timing(self._ctx, ctypes.byref(a), ctypes.byref(b)), "sv_get_last_bolt12_timing")
        return a.value, b.value

    def sha256_double(self, data, off, length):
        data = np.ascontiguousarray(data, dtype=np.uint8).reshape(-1)
        off = np.ascontiguousarray(off, dtype=np.uint64)
        length = np.ascontiguousarray(length, dtype=np.uint32)
        n = off.shape[0]
        out = np.zeros((n, 32), dtype=np.uint8)
        self._check(self.lib.sv_sha256d_host(self._ctx, data.ctypes.data, data.size, off.ctypes.data,
                                             length.ctypes.data, n, out.ctypes.data), "sv_sha256d_host")
        return out

    def pubkey_parse(self, key33):
        key33 = _u8(key33, 33)
        n = key33.shape[0]
        xy = np.zeros((n, 64), dtype=np.uint8)
        ok = np.zeros(n, dtype=np.uint8)
        self._check(self.lib.sv_pubkey_parse_host(self._ctx, key33.ctypes.data, n, xy.ctypes.data, ok.ctypes.data),
                    "sv_pubkey_parse_host")
        return xy, ok

    def verify_mixed(self, kinds, msg32, key64, sig64):
        """Interleaved batch: kinds (n,) uint8 SV_KIND_* tags, keys in 64-byte slots; verdicts in item order."""
        kinds = np.ascontiguousarray(kinds, dtype=np.uint8).reshape(-1)
        msg32, key64, sig64 = _u8(msg32, 32), _u8(key64, 64), _u8(sig64, 64)
        n = kinds.shape[0]
        out = np.zeros(max(n, 1), dtype=np.uint8)
        self._check(self.lib.sv_verify_mixed_host(self._ctx, kinds.ctypes.data, msg32.ctypes.data, key64.ctypes.data,
                                                  sig64.ctypes.data, n, out.ctypes.data), "sv_verify_mixed_host")
        return out[:n]

    def verify_schnorr_batch(self, msg32, xonly32, sig64, seed32=None):
        """BIP-340 batch verification (random linear combination per group of 1024, one-by-one for failed groups).
        Returns (verdicts, groups_total, groups_failed)."""
        msg32, xonly32, sig64 = _u8(msg32, 32), _u8(xonly32, 32), _u8(sig64, 64)
        n = msg32.shape[0]
        out = np.zeros(max(n, 1), dtype=np.uint8)
        gt, gf = ctypes.c_uint32(), ctypes.c_uint32()
        seed = np.ascontiguousarray(np.frombuffer(bytes(seed32), dtype=np.uint8)) if seed32 is not None else None
        self._check(self.lib.sv_verify_schnorr_batch_host(self._ctx, msg32.ctypes.data, xonly32.ctypes.data, sig64.ctypes.data, n,
                                                          seed.ctypes.data if seed is not None else None, out.ctypes.data,
                                                          ctypes.byref(gt), ctypes.byref(gf)), "sv_verify_schnorr_batch_host")
        return out[:n], gt.value, gf.value

    def set_dedup(self, on=True):
        self._check(self.lib.sv_set_dedup(self._ctx, 1 if on else 0), "sv_set_dedup")

    def set_nosqrt(self, on=True):
        """compressed-key ECDSA batches: the flow without the square root (default) or the plain one"""
        self._check(self.lib.sv_set_nosqrt(self._ctx, 1 if on else 0), "sv_set_nosqrt")

    def last_distinct_keys(self):
        return self.lib.sv_last_distinct_keys(self._ctx)

    def set_small_max(self, n):
        """largest batch that takes the small-batch (latency) path; 0 = always the throughput kernels"""
        self._check(self.lib.sv_set_small_max(self._ctx, int(n)), "sv_set_small_max")

    def small_max(self):
        return self.lib.sv_get_small_max(self._ctx)

    def selftest(self, op, a, b=None):
        """Run primitive `op` (SV_ST_* of cln_sigverify.h) of the device arithmetic on operands a, b: (n, 8) uint32
        little-endian limbs each; returns (n, 16) uint32.  Test support."""
        a = np.ascontiguousarray(a, dtype=np.uint32).reshape(-1, 8)
        b = np.zeros_like(a) if b is None else np.ascontiguousarray(b, dtype=np.uint32).reshape(-1, 8)
        if a.shape != b.shape:
            raise ValueError("operand shape mismatch")
        out = np.zeros((a.shape[0], 16), dtype=np.uint32)
        self._check(self.lib.sv_selftest_host(self._ctx, int(op), a.ctypes.data, b.ctypes.data, a.shape[0], out.ctypes.data),
                    "sv_selftest_host")
        return out

    def selftest_group(self, op, rec):
        """Run group op `op` (SV_STG_* of cln_sigverify.h) on the device for each record of rec: (n, 64) uint32; returns
        (n, 200) uint32.  Test support."""
        rec = np.ascontiguousarray(rec, dtype=np.uint32).reshape(-1, STG_IN_WORDS)
        out = np.zeros((rec.shape[0], STG_OUT_WORDS), dtype=np.uint32)
        self._check(self.lib.sv_selftest_group_host(self._ctx, int(op), rec.ctypes.data, rec.shape[0], out.ctypes.data),
                    "sv_selftest_group_host")
        return out

    # ---- deferral queue --------------------------------------------------------------------
    def enqueue(self, kind, msg32, key, sig64):
        m = np.ascontiguousarray(msg32, dtype=np.uint8)
        k = np.ascontiguousarray(key, dtype=np.uint8)
        s = np.ascontiguousarray(sig64, dtype=np.uint8)
        assert m.size == 32 and k.size == KEY_SIZE[kind] and s.size == 64
        idx = self.lib.sv_enqueue(self._ctx, kind, m.ctypes.data, k.ctypes.data, s.ctypes.data)
        if idx < 0:
            raise EngineError(f"sv_enqueue failed ({idx})")
        return idx

    def pending(self):
        return self.lib.sv_pending(self._ctx)

    def flush(self):
        n = self.pending()
        out = np.zeros(max(n, 1), dtype=np.uint8)
        self._check(self.lib.sv_flush(self._ctx, out.ctypes.data, n), "sv_flush")
        return out[:n]

    # ---- device-buffer API (pointers: ints, e.g. torch tensor .data_ptr()) -----------------
    def verify_device(self, kind, d_msg, d_key, d_sig, n, d_verdict, d_bitmap=0, stream=0):
        self._check(self.lib.sv_verify_device(self._ctx, kind, d_msg, d_key, d_sig, n, d_verdict, d_bitmap or None,
                                              stream or None), "sv_verify_device")

    def synth_device(self, kind, seed, n, d_msg, d_key, d_sig, stream=0):
        self._check(self.lib.sv_synth_device(self._ctx, kind, seed, n, d_msg, d_key, d_sig, stream or None),
                    "sv_synth_device")

    def stream_handle(self):
        """cudaStream_t of the context's own stream (wrap with torch.cuda.ExternalStream to time on it)."""
        return self.lib.sv_get_stream(self._ctx)

    def sync(self, stream=0):
        self._check(self.lib.sv_sync(self._ctx, stream or None), "sv_sync")

    def set_profiling(self, on=True):
        self._check(self.lib.sv_set_profiling(self._ctx, 1 if on else 0), "sv_set_profiling")

    def last_timing(self):
        """(prep_ms, main_ms) device time of the last verify launch pair; call after sync()."""
        a, b = ctypes.c_float(), ctypes.c_float()
        self._check(self.lib.sv_get_last_timing(self._ctx, ctypes.byref(a), ctypes.byref(b)), "sv_get_last_timing")
        return a.value, b.value

    def host_alloc(self, nbytes):
        """Pinned host buffer as a numpy uint8 array (cudaHostAlloc); free with host_free(arr)."""
        p = self.lib.sv_host_alloc(nbytes)
        if not p:
            raise EngineError("sv_host_alloc failed")
        buf = (ctypes.c_uint8 * nbytes).from_address(p)
        arr = np.frombuffer(buf, dtype=np.uint8)
        self._pinned = getattr(self, "_pinned", {})
        self._pinned[arr.ctypes.data] = p
        return arr

    def host_free(self, arr):
        p = getattr(self, "_pinned", {}).pop(arr.ctypes.data, None)
        if p:
            self.lib.sv_host_free(p)

    def info(self):
        inf = SvInfo()
        self._check(self.lib.sv_get_info(self._ctx, ctypes.byref(inf)), "sv_get_info")
        return {f[0]: getattr(inf, f[0]) for f in SvInfo._fields_}

    def probe(self, mode):
        v = ctypes.c_double()
        self._check(self.lib.sv_probe(self._ctx, mode, ctypes.byref(v)), "sv_probe")
        return v.value
