"""GPU replay of tests/golden/keyed_plans.npz: every keyed call of tests/keyed_plan_cases.py, under the budget of each of its plans
(resident in one chunk, resident in several chunks, streamed in one key range, streamed through several), records the key bounds
and the streamed flag the fixture holds and computes its outputs: scoring and one-row-key fits bit for bit, other fits within the
run-to-run spread of the CSR kernels' float-atomic gradient sums."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import keyed_plan_cases as kc  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "keyed_plans.npz")


@pytest.fixture(scope="module")
def keyed_plans():
    return np.load(GOLDEN)


@pytest.mark.parametrize("name", list(kc.CASES))
def test_keyed_call_keeps_its_plans_and_outputs(keyed_plans, name):
    import mlease_b200 as mb
    data = kc.CASES[name]["make"]()
    bitwise = kc.CASES[name].get("bitwise", False)
    plans = kc.CASES[name].get("plans", ("resident", "chunked", "streamed"))
    for i in range(len(plans)):
        key = "%s__%d__" % (name, i)
        budget = int(keyed_plans[key + "budget"])
        bounds, streamed, out = kc.run(mb, name, budget, data)
        assert np.array_equal(bounds, keyed_plans[key + "bounds"]), (budget, bounds, keyed_plans[key + "bounds"])
        assert streamed == bool(keyed_plans[key + "streamed"]), budget
        assert set(out) == {k[len(key):] for k in keyed_plans.files if k.startswith(key)} - {"budget", "bounds", "streamed"}
        for k, got in out.items():
            want = keyed_plans[key + k]
            assert got.shape == want.shape and got.dtype == want.dtype, (budget, k)
            if bitwise or got.dtype != np.float64:
                assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), (budget, k)
            else:
                assert np.all(np.abs(got - want) <= 1e-6 * np.maximum(1.0, np.abs(want))), (budget, k)
