"""CPU: the verifier subdaemon's BOLT12 messages (sigverifyd_bolt12 / sigverifyd_bolt12_reply) at the shapes the feature
sends: empty streams, long streams, with and without sighashes.  The generated C codec and the generated Python codec must
agree byte for byte in both directions, and both must refuse truncated frames, counts that do not match the bytes that
follow and a message of another type (tests/sigverifyd_codec.py)."""
import numpy as np
import pytest

from tests import sigverifyd_codec as codec

RID = 0x0102030405060708


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    return codec.build_shim(tmp_path_factory.mktemp("wire"))


def _request(rng, lens, want):
    n = len(lens)
    blob = rng.integers(0, 256, size=sum(lens), dtype=np.uint8).tobytes()
    xonly = rng.integers(0, 256, size=32 * n, dtype=np.uint8).tobytes()
    sigs = rng.integers(0, 256, size=64 * n, dtype=np.uint8).tobytes()
    return dict(req_id=RID, mnlen=15, messagename=b"invoice_request", fnlen=9, fieldname=b"signature", n=n, lens=lens,
                bloblen=len(blob), blob=blob, xonly=xonly, sigs=sigs, want_sighash=want)


@pytest.mark.parametrize("lens", [[], [0], [0, 300, 0], [20_001], [5, 20_500, 1, 0, 77]],
                         ids=["n0", "empty_stream", "empty_among_others", "long_stream", "mixed"])
@pytest.mark.parametrize("want", [0, 1], ids=["no_sighash", "want_sighash"])
def test_request_codecs_agree(shim, lens, want):
    req = _request(np.random.default_rng(len(lens) * 10 + want), lens, want)
    codec.agree(shim, "sigverifyd_bolt12", req)
    codec.refused(shim, "sigverifyd_bolt12", req)


@pytest.mark.parametrize("n", [0, 1, 7, 25_000])
@pytest.mark.parametrize("want", [0, 1], ids=["no_sighash", "want_sighash"])
def test_reply_codecs_agree(shim, n, want):
    rng = np.random.default_rng(n + want)
    status = bytes(rng.choice([0, 1, 255], size=n).astype(np.uint8))
    nsh = n if want else 0
    sh = rng.integers(0, 256, size=32 * nsh, dtype=np.uint8).tobytes()
    rep = dict(req_id=RID, n=n, status=status, nsighash=nsh, sighashes=sh)
    codec.agree(shim, "sigverifyd_bolt12_reply", rep)
    codec.refused(shim, "sigverifyd_bolt12_reply", rep)


def test_wrong_type_is_refused(shim):
    codec.wrong_type_refused(shim, "sigverifyd_bolt12", _request(np.random.default_rng(3), [4], 1))
    rep = dict(req_id=RID, n=1, status=b"\x01", nsighash=0, sighashes=b"")
    codec.wrong_type_refused(shim, "sigverifyd_bolt12_reply", rep)
