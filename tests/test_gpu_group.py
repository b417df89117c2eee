"""GPU: the group law and the multiplication schedules on the device, and the constructed exceptional-addition fixture
through every verification route.

The group self-test ops (tests/group_cases.py) run through sv_selftest_group_host -> k_selftest_group at full size: about
10^5 records per point operation, thousands per schedule, plus the crafted ladder and comb inputs.  The fixture
tests/golden/group_exceptional.npz (tests/group_fixture.py) goes through each route that selects a different schedule;
every verdict must equal the reference's, stored with the fixture and checked against the recorded reference by
tests/test_group_emul.py.  Hit counts go to $SV_SELFTEST_COVERAGE_DIR/group_coverage.json when that is set."""
import json
import os

import numpy as np
import pytest

from tests import group_cases as C
from tests import group_fixture as F
from tests.test_group_emul import coverage, crafted_combs, crafted_ladders

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _coverage():
    C.COVERAGE.clear()
    yield
    out = os.environ.get("SV_SELFTEST_COVERAGE_DIR")
    if out:
        os.makedirs(out, exist_ok=True)
        sched = {k: {f"{s}.{b}": n for (s, b), n in sorted(v.items())} for k, v in sorted(coverage().items())}
        with open(os.path.join(out, "group_coverage.json"), "w") as f:
            json.dump({"ops": dict(sorted(C.COVERAGE.items())), "schedules": sched, "routes": ROUTES}, f, indent=1)


ROUTES = {}


def test_group_point_ops(engine):
    C.case_gej_double(engine)
    C.case_gej_add_ge(engine)
    C.case_gej_add_gej(engine)
    C.case_ge_set_xo(engine)


def test_group_tables_ladders_combs_linear_form(engine):
    C.case_qtable_build(engine)
    C.case_ladders(engine, crafted=crafted_ladders())
    C.case_combs(engine, crafted=crafted_combs())
    C.case_ns_linear_form(engine)


def _sets():
    fx = F.load()
    return fx, ((0, fx["ecdsa_msg"], fx["ecdsa_pub33"], fx["ecdsa_sig"]),
                (1, fx["ecdsa_msg"], fx["ecdsa_pubxy"], fx["ecdsa_sig"]),
                (2, fx["bip340_msg"], fx["bip340_xonly"], fx["bip340_sig"]))


def _tile(a, n):
    return np.concatenate([a] * (n // a.shape[0] + 1))[:n]


def test_constructed_fixture_through_every_route(engine):
    import torch
    fx, sets = _sets()
    sm = engine.small_max()
    try:
        for kind, msg, key, sig in sets:
            want = fx[f"ref_verdict_{kind}"]
            n = msg.shape[0]
            for nosqrt in (True, False):
                engine.set_nosqrt(nosqrt)
                # small-batch kernel (whole fixture at or below small_max) and throughput kernels (small_max 0)
                for limit, name in ((max(n, sm), "small"), (0, "throughput")):
                    engine.set_small_max(limit)
                    got = engine.verify(kind, msg, key, sig)
                    assert np.array_equal(got, want), (kind, nosqrt, name, np.nonzero(got != want)[0])
                    ROUTES[f"verify.kind{kind}.{name}.nosqrt{int(nosqrt)}"] = n
                # above small_max at the default threshold: the fixture tiled past it
                engine.set_small_max(sm)
                m = sm + 1 + n
                got = engine.verify(kind, _tile(msg, m), _tile(key, m), _tile(sig, m))
                assert np.array_equal(got, _tile(want, m)), (kind, nosqrt, "tiled")
                # on the device: caller arrays, verdicts in device memory
                d = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (msg, key, sig)]
                out = torch.zeros(n, dtype=torch.uint8, device="cuda")
                torch.cuda.synchronize()
                engine.verify_device(kind, d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), n, out.data_ptr())
                engine.sync()
                assert np.array_equal(out.cpu().numpy(), want), (kind, nosqrt, "verify_device")
                ROUTES[f"verify_device.kind{kind}.nosqrt{int(nosqrt)}"] = n
            engine.set_nosqrt(True)
            if kind != 2:  # one key per item: the shared-key path
                for i in range(n):
                    got = engine.verify_samekey(kind, key[i], msg[i:i + 1], sig[i:i + 1])
                    assert got[0] == want[i], (kind, i, "samekey")
                ROUTES[f"samekey.kind{kind}"] = n
            for i in range(n):
                engine.enqueue(kind, msg[i], key[i], sig[i])
            got = engine.flush()
            assert np.array_equal(np.asarray(got)[:n], want), (kind, "enqueue/flush")
            ROUTES[f"flush.kind{kind}"] = n
        # all three kinds interleaved in one batch
        kinds, msgs, keys, sigs, wants = [], [], [], [], []
        for kind, msg, key, sig in sets:
            k64 = np.zeros((msg.shape[0], 64), np.uint8)
            k64[:, :key.shape[1]] = key
            kinds.append(np.full(msg.shape[0], kind, np.uint8))
            msgs.append(msg)
            keys.append(k64)
            sigs.append(sig)
            wants.append(fx[f"ref_verdict_{kind}"])
        order = np.random.default_rng(5).permutation(sum(len(k) for k in kinds))
        cat = lambda xs: np.concatenate(xs)[order]
        for limit in (0, sm):
            engine.set_small_max(limit)
            got = engine.verify_mixed(cat(kinds), cat(msgs), cat(keys), cat(sigs))
            assert np.array_equal(got, cat(wants)), ("mixed", limit)
            ROUTES[f"mixed.small_max{limit}"] = len(order)
    finally:
        engine.set_small_max(sm)
        engine.set_nosqrt(True)
