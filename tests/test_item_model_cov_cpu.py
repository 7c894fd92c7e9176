"""CPU checks of the host side of item_model_train_cov: the exact list lengths the wrapper allocates from, the (prior, key) order of
keyed_cov_for_scoring, and the packed lower-triangle layout the tests read the blocks with."""
import numpy as np

import item_model_cov_ref as ref


def test_list_lengths_count_each_keys_distinct_columns():
    from mlease_b200.admm import _list_lengths
    krs = np.array([0, 2, 2, 5], np.int64)   # key 1 has no rows
    rp = np.array([0, 3, 5, 6, 8, 10], np.int64)
    ci = np.array([1, 4, 7, 4, 9, 0, 0, 3, 3, 8], np.int32)
    assert list(_list_lengths(krs, rp, ci, 10)) == [4 + 1, 0, 3 + 1]


def test_keyed_cov_for_scoring_orders_blocks_by_prior_then_key():
    from mlease_b200 import keyed_cov_for_scoring, keyed_models_for_scoring
    key_ptr = np.array([0, 2, 2, 5], np.int64)
    n = np.diff(key_ptr)
    cov_ptr = np.concatenate([[0], np.cumsum(n * (n + 1) // 2)]).astype(np.int64)
    m = int(cov_ptr[-1])
    cov = np.arange(2 * 3 * m, dtype=np.float64).reshape(2, 3, m)
    ptrs, vals = keyed_cov_for_scoring(key_ptr, cov_ptr, cov)
    mp, _, _ = keyed_models_for_scoring(key_ptr, np.arange(5), np.zeros((2, 3, 5)))
    assert len(ptrs) == len(mp) == 6 * 3 + 1
    for p in range(6):
        for k in range(3):
            got = vals[ptrs[p * 3 + k]:ptrs[p * 3 + k + 1]]
            assert np.array_equal(got, cov.reshape(6, m)[p, cov_ptr[k]:cov_ptr[k + 1]])
            nm = mp[p * 3 + k + 1] - mp[p * 3 + k]
            assert len(got) == nm * (nm + 1) // 2


def test_packed_layout_and_reference_inverse():
    rng = np.random.default_rng(5)
    A = rng.normal(size=(6, 6))
    H = A @ A.T + 6 * np.eye(6)
    S, kappa = ref.inverse(H)
    assert np.allclose(S @ H, np.eye(6), atol=1e-12) and kappa >= 1
    block = np.array([S[a, b] for a in range(6) for b in range(a + 1)])
    assert np.array_equal(ref.unpack(block, 6), np.tril(S) + np.tril(S, -1).T)
