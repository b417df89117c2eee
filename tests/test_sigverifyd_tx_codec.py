"""CPU: the verifier subdaemon's transaction messages (sigverifyd_tx / sigverifyd_tx_reply) at the shapes the feature
sends: both key kinds, with and without sighashes, a 70,000-byte span, up to 65,536 replies.  The generated C codec and the
generated Python codec must agree byte for byte in both directions, and both must refuse truncated and over-long frames,
counts that do not match the bytes that follow, and the wrong message type (tests/sigverifyd_codec.py)."""
import numpy as np
import pytest

from tests import sigverifyd_codec as codec

RID = 0x0102030405060708
U32_ARRAYS = ["version", "locktime", "sequence", "sighash_type", "prev_index", "flags"]
LEN_ARRAYS = ["script_len", "outputs_len", "prevouts_len", "sequences_len"]


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    return codec.build_shim(tmp_path_factory.mktemp("wire"))


def _request(rng, n, kind, want):
    """a request of n transactions with random field values (the codec does not care what they mean)"""
    ks = 33 if kind == 0 else 64
    req = dict(req_id=RID, kind=kind, keylen=ks, key=rng.integers(0, 256, size=ks, dtype=np.uint8).tobytes(), n=n)
    for f in U32_ARRAYS:
        req[f] = [int(x) for x in rng.integers(0, 2**32, size=n, dtype=np.uint64)]
    req["prev_txid"] = rng.integers(0, 256, size=32 * n, dtype=np.uint8).tobytes()
    for f in ("input_amount", "output_amount"):
        req[f] = [int(x) for x in rng.integers(0, 2**63, size=n, dtype=np.uint64)] if n else []
    for f in LEN_ARRAYS:
        req[f] = [int(x) for x in rng.integers(0, 300, size=n)]
    if n:
        req["script_len"][0] = 70_000  # one long span
    total = sum(sum(req[f]) for f in LEN_ARRAYS)
    req.update(bloblen=total, blob=rng.integers(0, 256, size=total, dtype=np.uint8).tobytes(),
               sigs=rng.integers(0, 256, size=64 * n, dtype=np.uint8).tobytes(), want_sighash=want)
    return req


def _reply(rng, n, want):
    nsh = n if want else 0
    return dict(req_id=RID, n=n, verdicts=bytes(rng.integers(0, 2, size=n).astype(np.uint8)), nsighash=nsh,
                sighashes=rng.integers(0, 256, size=32 * nsh, dtype=np.uint8).tobytes())


@pytest.mark.parametrize("n", [0, 1, 3, 483])
@pytest.mark.parametrize("kind", [0, 1], ids=["ecdsa33", "ecdsa_xy"])
@pytest.mark.parametrize("want", [0, 1], ids=["no_sighash", "want_sighash"])
def test_request_codecs_agree(shim, n, kind, want):
    req = _request(np.random.default_rng(n * 4 + kind * 2 + want), n, kind, want)
    codec.agree(shim, "sigverifyd_tx", req)
    codec.refused(shim, "sigverifyd_tx", req)


@pytest.mark.parametrize("n", [0, 1, 7, 484, 65_536])
@pytest.mark.parametrize("want", [0, 1], ids=["no_sighash", "want_sighash"])
def test_reply_codecs_agree(shim, n, want):
    rep = _reply(np.random.default_rng(n + want), n, want)
    codec.agree(shim, "sigverifyd_tx_reply", rep)
    codec.refused(shim, "sigverifyd_tx_reply", rep)


def test_wrong_type_is_refused(shim):
    rng = np.random.default_rng(3)
    codec.wrong_type_refused(shim, "sigverifyd_tx", _request(rng, 2, 1, 1))
    codec.wrong_type_refused(shim, "sigverifyd_tx_reply", _reply(rng, 2, 0))
