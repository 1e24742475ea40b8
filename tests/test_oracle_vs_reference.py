"""Differential test: the numpy oracle against results of the UNMODIFIED reference on seeds that were NOT screened
for unambiguous ReLU gates (oracle/cases.py UNSCREENED).  The reference's results are stored vectors
(tests/golden/unscreened_*.npz, gather_random_users.npz; oracle/make_golden.py writes them)."""
import numpy as np
import pytest

from oracle import cases as C
from oracle import recnn_oracle as O
from tests._golden import compare_with_golden, load_golden, run_oracle_case


@pytest.mark.parametrize("opt", ["adam", "sgd"])
@pytest.mark.parametrize("algo", ["ddpg", "td3"])
@pytest.mark.parametrize("spec", list(C.UNSCREENED.values()), ids=list(C.UNSCREENED))
def test_oracle_tracks_the_live_reference(spec, algo, opt):
    cid = next(k for k, v in C.UNSCREENED.items() if v is spec)
    ref = load_golden("unscreened_%s_%s_%s.npz" % (cid, algo, opt))
    if float(ref["gate_margin"]) <= C.GATE_GUARD:
        pytest.skip("unscreened seed with an ambiguous ReLU gate (margin %.2g): torch/MKL and numpy may gate "
                    "differently; the screened golden seeds cover this algorithm" % float(ref["gate_margin"]))
    got = run_oracle_case(spec, algo, opt, golden=ref if algo == "td3" else None)
    compare_with_golden(got, ref, check_grads=(algo == "ddpg"))


def test_reference_gather_equals_oracle_on_random_users():
    ref = load_golden("gather_random_users.npz")
    frame = int(ref["frame_size"])
    users = []
    i = 0
    while "user%d.items" % i in ref:
        items = ref["user%d.items" % i]
        users.append({"items": items, "rates": ref["user%d.rates" % i], "sizes": len(items),
                      "users": int(ref["user%d.id" % i])})
        i += 1
    assert len(users) == 5
    col = O.collate_users(users, frame)
    out = O.frame_gather(ref["table"], col["items"], col["ratings"], col["sizes"], frame)
    for k in ("state", "next_state", "action", "reward", "done"):
        assert np.array_equal(out[k].view(np.uint32), ref["out." + k].view(np.uint32)), k
