"""Host build: the signatures of tests/golden/invalid_curve.npz, forged for 64-byte keys off secp256k1, are refused, and
each would be accepted if one key gate were gone.

The construction is rechecked with Python integers (the key is off secp256k1 and of order h on its own curve, r is the x
of j*Q, the device's ladder lands on j*Q).  The unmodified host build refuses every case on every entry point that takes
a 64-byte key.  Then, for each of the four places that keep a key's decode flag in the verdict, a copy of the kernel
source without that one gate is built for the host and must accept the cases on the entry points that run it: the
evidence that the cases reach the gate, so that the device tests of tests/test_gpu_invalid_curve.py can tell a dropped
gate from a working one."""
import ctypes
import random
import shutil

import numpy as np
import pytest

from lightning_b200 import build
from tests import ecc
from tests import invalid_curve as I
from tests.limb_model import split_lambda

N = I.N


@pytest.fixture(scope="module")
def fx():
    return I.load()


@pytest.fixture(scope="session")
def mutant_libs(tmp_path_factory):
    """{gate name: host build without that gate}, built once per session"""
    tmp = str(tmp_path_factory.mktemp("invalid_curve_mutants"))
    return {name: ctypes.CDLL(I.build_mutant(name, tmp)) for name in I.MUTANTS}


def _int(b):
    return int.from_bytes(bytes(b), "big")


def test_fixture_is_the_construction(fx):
    """the committed cases are what tests/invalid_curve.py builds today (the classes and subgroups checked on the way),
    and the reference refused every one when they were generated"""
    built = I.build_cases()
    for k, v in built.items():
        assert np.array_equal(fx[k], v), k
    assert fx["ref_verdict"].shape == (fx["msg"].shape[0],) and not fx["ref_verdict"].any()
    assert not fx["emul_verdict"].any()
    assert list(fx["mutant"]) == sorted(I.MUTANTS) and fx["mutant_verdict"].all()
    per_class = {b: int((fx["b"] == b).sum()) for b in (2, 4, 6, 3)}
    assert set(fx["b"].tolist()) == {2, 4, 6, 3} and min(per_class.values()) >= 2, per_class


def test_construction_with_python_integers(fx):
    """per case: Q off secp256k1, on y^2 = x^3 + b with exact order h (h prime); r = x(j*Q) < n, 0 < s <= n/2, the
    message reduces to 0 mod n; the device's ladder (forced-odd GLV halves, 4-bit windows over {1, 3, ..., 15}*Q, phi on
    the second half) computes u2*Q = j*Q with u2 = r/s; and a plain GLV split without the forcing would not always
    predict it.  Every key carries several distinct s."""
    naive_wrong = 0
    for g in np.unique(fx["group"]):
        sel = np.nonzero(fx["group"] == g)[0]
        b, h = int(fx["b"][sel[0]]), int(fx["h"][sel[0]])
        assert (fx["b"][sel] == b).all() and (fx["h"][sel] == h).all() and (fx["key"][sel] == fx["key"][sel[0]]).all()
        assert all(h % q for q in range(2, int(h ** 0.5) + 1)) and h % 3 == 1
        Q = (_int(fx["key"][sel[0], :32]), _int(fx["key"][sel[0], 32:]))
        assert Q[0] < I.P and Q[1] < I.P
        assert I.on_curve(Q, b) and not I.on_curve(Q, 7)
        assert Q is not None and I.mul(h, Q) is None
        mu = I.eigenvalue(Q, h)
        sigs = {bytes(fx["sig"][i]) for i in sel}
        assert len(sigs) == I.SIGS_PER_KEY, (b, h, len(sigs))
        for i in sel:
            r, s, j = _int(fx["sig"][i, :32]), _int(fx["sig"][i, 32:]), int(fx["j"][i])
            assert _int(fx["msg"][i]) % N == 0
            assert 0 < r < N and 0 < s <= N // 2
            R = I.mul(j, Q)
            assert R is not None and R[0] == r
            u2 = r * pow(s, -1, N) % N
            assert I.predict(u2, mu, h) == j
            assert I.ladder_point(u2, Q) == R, (b, h, i)
            k1, k2 = (k - N if k > N // 2 else k for k in split_lambda(u2))
            naive_wrong += (k1 + mu * k2) % h != j
    assert naive_wrong > 0  # the forcing to odd halves matters for the prediction


def test_unmodified_host_build_refuses_every_case(fx, emul):
    """kind 1 through the throughput path, the small-batch path (sequential and on lane pairs) and the shared-key path:
    every verdict 0; and the same items beside valid 64-byte-key signatures leave those valid"""
    for route in I.ROUTES:
        got = I.run_route(emul, route, fx)
        assert not got.any(), (route, np.nonzero(got)[0])
    # among valid signatures, at the edges of a 32-item inversion batch
    rng = random.Random("invalid-curve/host-bg")
    n = 70
    msg = np.zeros((n, 32), np.uint8)
    key = np.zeros((n, 64), np.uint8)
    sig = np.zeros((n, 64), np.uint8)
    want = np.ones(n, np.uint8)
    for i in range(n):
        sk = rng.randrange(1, N).to_bytes(32, "big")
        m = rng.randbytes(32)
        msg[i], key[i], sig[i] = (np.frombuffer(v, np.uint8) for v in (m, ecc.pubkey_create(sk)[1], ecc.ecdsa_sign(sk, m)))
    pos = [0, 15, 16, 31, 32, 33, 47, n - 1]
    for c, p in enumerate(pos):
        i = (7 * c) % fx["msg"].shape[0]
        msg[p], key[p], sig[p], want[p] = fx["msg"][i], fx["key"][i], fx["sig"][i], 0
    for route in ("emul_verify_batch", "emul_verify_small_batch", "emul_verify_small_pair_batch"):
        out = np.zeros(n, np.uint8)
        getattr(emul, route)(1, I.ptr(msg), I.ptr(key), I.ptr(sig), ctypes.c_size_t(n), I.ptr(out))
        assert np.array_equal(out, want), (route, np.nonzero(out != want)[0])


@pytest.mark.parametrize("gate", sorted(I.MUTANTS))
def test_each_gate_is_what_refuses(fx, emul, mutant_libs, gate):
    """the host build without `gate` accepts every case on each entry point that runs the gate, where the unmodified build
    refuses the same bytes; entry points that do not run it still refuse.  The stored verdicts of the fixture agree."""
    lib = mutant_libs[gate]
    routes = I.MUTANTS[gate][3]
    counts = {}
    for route in I.ROUTES:
        got = I.run_route(lib, route, fx)
        base = I.run_route(emul, route, fx)
        assert not base.any(), route
        if route in routes:
            counts[route] = int(got.sum())
            assert got.all(), (gate, route, f"{int(got.sum())} of {got.size} accepted", np.nonzero(got == 0)[0][:8])
        else:
            assert not got.any(), (gate, route, "accepts without running the gate")
    col = list(fx["mutant"]).index(gate)
    assert np.array_equal(fx["mutant_verdict"][:, col], I.run_route(lib, routes[0], fx)), gate
    print(f"without {gate}: " + ", ".join(f"{r} accepts {c} of {fx['msg'].shape[0]}" for r, c in counts.items()))


def test_a_gate_that_moved_fails_loudly(tmp_path):
    """build_mutant refuses a source where the gate's text is gone or occurs twice"""
    csrc = tmp_path / "csrc"
    shutil.copytree(build.CSRC, csrc)
    fname, gate, _, _ = I.MUTANTS["verify_curve_side"]
    text = (csrc / fname).read_text()
    for changed in (text.replace(gate, gate.replace("kd", "key_ok_")), text.replace(gate, gate + gate)):
        (csrc / fname).write_text(changed)
        with pytest.raises(AssertionError, match="occurs"):
            I.build_mutant("verify_curve_side", str(tmp_path / "w"), csrc=str(csrc))
