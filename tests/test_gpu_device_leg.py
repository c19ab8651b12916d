"""GPU tests of the device leg's repair check (EmbedScorer.recommend_device_async / _Pending.result): the
count of rows with a non-zero status that b200_recommend_embed copies to a pinned word after each launch.

A catalogue with 4 001 identical item rows and 500 users aligned with them: those users' candidate sets
are far too tied for the fused path, so their rows are flagged (and so are other users' rows whose top-K
reaches the tied items).  Two calls are
kept in flight as a server (and bench.py's device leg) does: the first has 40 000 users, so two launches
write one count each, and its handle is checked only after the second call is enqueued.  Each handle must
report exactly the rows its own call flagged, and return the exact path's ids after the repair.
"""
import numpy as np
import pytest

from test_gpu_fused_c2 import _tables

pytestmark = pytest.mark.gpu


def test_flagged_rows_of_two_calls_in_flight():
    import torch
    from librecommender_b200.engine import FUSED_ROWS_PER_CALL, EmbedScorer

    n_users, N, d, K = 50_000, 300_003, 64, 50
    U, I = _tables(81, n_users, N, d)
    I[1:4001] = I[0]
    U[:500] = I[0]
    sc = EmbedScorer(U, I, N, None, n_users=n_users)
    rng = np.random.default_rng(82)
    rest = rng.permutation(np.arange(500, n_users))
    hot = rng.permutation(500)
    calls = [np.concatenate([hot[:150], rest[:39_700], hot[150:300]]),   # tied users in both launches
             np.concatenate([rest[39_700:49_000], hot[300:]])]
    assert len(calls[0]) > FUSED_ROWS_PER_CALL
    uids = [torch.as_tensor(c.astype(np.int64)).cuda() for c in calls]

    flagged = []
    for uid in uids:
        status = sc.recommend_fused(uid, K, False, False)[2].cpu().numpy()
        flagged.append(int((status != 0).sum()))
    assert flagged[0] >= 300 and flagged[1] >= 200, flagged

    pending = [sc.recommend_device_async(uid, K, False, False) for uid in uids]
    for p, uid, n_bad in zip(pending, uids, flagged):
        ids = p.result()
        assert sc.last_fallback_rows == n_bad
        exact = sc.recommend_exact(uid, K, False, False)
        np.testing.assert_array_equal(ids.cpu().numpy(), exact.cpu().numpy())
