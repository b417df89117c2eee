"""Generate tests/golden/invalid_curve.npz: ECDSA signatures forged for 64-byte keys off secp256k1 (tests/invalid_curve.py),
with the verdicts of the reference and of host builds that each lack one key gate.

Needs oracle/_ref/libsecp_ref.so (oracle/Makefile, from a Core Lightning source tree) and g++.  Deterministic: the same
file on every run.

Arrays (n cases): b (the curve y^2 = x^3 + b of the key), h (the key's order on it), j (r = x(j*Q), and u2*Q == j*Q as the
engine computes it), group (cases of one key share it), key (n, 64: x || y), sig (n, 64: r || s), msg (n, 32: zero, or
the encoding of n), ref_verdict (the reference: secp256k1_ec_pubkey_parse(04 || x || y) then verify; 0 for every case),
emul_verdict (the unmodified host build, emul_verify_batch: 0), mutant (names of the gates, tests.invalid_curve.MUTANTS),
mutant_verdict (n, len(mutant): the host build without that gate, on the first entry point that runs it).
Run:  python -m tests.golden.make_invalid_curve
"""
import ctypes
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tests import invalid_curve as I, util  # noqa: E402
from tests.golden.make_bip143_sweep import save  # noqa: E402


def main():
    fx = I.build_cases()
    n = fx["msg"].shape[0]
    fx["ref_verdict"] = util.ref_verify(util.load_ref(), 1, fx["msg"], fx["key"], fx["sig"])
    assert not fx["ref_verdict"].any(), "the reference accepts a key off the curve"
    fx["emul_verdict"] = I.run_route(util.load_emul(), "emul_verify_batch", fx)
    assert not fx["emul_verdict"].any(), "the host build accepts a forged signature"
    names = sorted(I.MUTANTS)
    fx["mutant"] = np.array(names)
    fx["mutant_verdict"] = np.zeros((n, len(names)), np.uint8)
    with tempfile.TemporaryDirectory() as tmp:
        for i, name in enumerate(names):
            lib = ctypes.CDLL(I.build_mutant(name, tmp))
            fx["mutant_verdict"][:, i] = I.run_route(lib, I.MUTANTS[name][3][0], fx)
    save(I.FIXTURE, fx)
    per = ", ".join(f"{name} {int(fx['mutant_verdict'][:, i].sum())}" for i, name in enumerate(names))
    print(f"{n} cases on {len(np.unique(fx['group']))} keys; accepted without the gate: {per}; "
          f"{os.path.getsize(I.FIXTURE)} bytes")


if __name__ == "__main__":
    main()
