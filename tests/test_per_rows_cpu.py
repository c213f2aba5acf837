"""Host-side rules of prioritised replay beyond 4096 rows: the uniform stream of the captured prioritised epoch, a NumPy
statement of the two-level search of trl_per_sample_rows, the ring-size refusal and the entry points' refusals."""
import ctypes

import numpy as np
import pytest

from tests.test_data_path_kernels import _buf16
from tests.test_layer_kernels import _rejects

CHUNK = 4096


def test_one_draw_of_all_uniforms_is_the_per_update_stream():
    """update_per_epoch draws rand(U * b) once; the eager loop it replaced drew rand(b) U times"""
    U, b = 13, 64
    np.random.seed(7)
    whole = np.random.rand(U * b)
    np.random.seed(7)
    parts = np.concatenate([np.random.rand(b) for _ in range(U)])
    assert np.array_equal(whole, parts)


def two_level_search(p, targets, chunk=CHUNK):
    """trl_per_sample_rows' rule in NumPy: in-chunk prefixes, chunk offsets, the global prefix fl(offset + local),
    the chunk found through the running maximum of each chunk's last global prefix (the last chunk if none exceeds
    the target), then the row inside it (its last row if none does); a zero-priority answer moves to the next positive
    row, else to the last positive row."""
    p = np.asarray(p, dtype=np.float64)
    n = len(p)
    starts = np.arange(0, n, chunk)
    local = np.concatenate([np.cumsum(p[s:s + chunk]) for s in starts])
    totals = np.array([local[min(s + chunk, n) - 1] for s in starts])
    offsets = np.concatenate([[0.0], np.cumsum(totals)[:-1]])
    glob = np.concatenate([offsets[c] + local[s:s + chunk] for c, s in enumerate(starts)])
    ends = np.maximum.accumulate(np.array([glob[min(s + chunk, n) - 1] for s in starts]))
    positive = np.flatnonzero(p > 0)
    out = []
    for t in targets:
        c = min(int(np.searchsorted(ends, t, side="right")), len(starts) - 1)
        s, e = starts[c], min(starts[c] + chunk, n)
        a = min(s + int(np.searchsorted(glob[s:e], t, side="right")), e - 1)
        later = positive[positive >= a]
        out.append(later[0] if later.size else positive[-1])
    return np.array(out), glob


@pytest.mark.parametrize("layout", ["plain", "zero_chunks", "boundary", "trailing"])
def test_two_level_search_equals_one_search_on_the_global_prefix(layout):
    rs = np.random.RandomState(1)
    n = 5 * CHUNK + 77
    p = rs.randint(0, 1025, n) * 2.0 ** -10
    if layout == "zero_chunks":
        p[CHUNK:3 * CHUNK] = 0.0
    elif layout == "boundary":
        for c in range(1, 6):
            p[c * CHUNK - 2:c * CHUNK + 3] = 0.0
    elif layout == "trailing":
        p[-CHUNK - 9:] = 0.0
    b = 2048
    u = rs.rand(b)
    u[-1] = 1.0 - 2.0 ** -53
    u[0] = 0.0
    glob_total = np.cumsum(p)[-1]
    targets = (np.arange(b) + u) / b * glob_total
    got, glob = two_level_search(p, targets)
    assert np.array_equal(glob, np.cumsum(p))              # exact regime: the two-level prefix is np.cumsum
    want = np.minimum(np.searchsorted(np.cumsum(p), targets, side="right"), np.flatnonzero(p > 0)[-1])
    assert np.array_equal(got, want)
    assert np.all(p[got] > 0)
    # chunk-boundary targets: exactly at each chunk's end, and just below it
    edges = np.cumsum(p)[np.arange(CHUNK - 1, n, CHUNK)]
    for t in np.concatenate([edges, np.nextafter(edges, 0)]):
        g, _ = two_level_search(p, [t])
        w = min(np.searchsorted(np.cumsum(p), t, side="right"), np.flatnonzero(p > 0)[-1])
        if p[w] == 0:
            w = np.flatnonzero(p > 0)[np.flatnonzero(p > 0) >= w][0]
        assert g[0] == w


def test_construction_refuses_rings_over_2_to_the_24_rows():
    from torchrl_b200.replay_buffers import PrioritizedReplayBuffer
    PrioritizedReplayBuffer((1 << 24) * 2, env_nums=2)                    # exactly 2^24 rows: accepted (lazy storage)
    with pytest.raises(ValueError, match="holds 1..16777216 time rows"):
        PrioritizedReplayBuffer((1 << 24) + 1)
    with pytest.raises(ValueError):
        PrioritizedReplayBuffer(3, env_nums=4)                            # zero rows


def test_new_entry_points_reject_bad_arguments(native_lib):
    buf, p = _buf16()
    L = native_lib
    assert L.trl_per_scratch_doubles(0) == -1 and L.trl_per_scratch_doubles((1 << 24) + 1) == -1
    assert L.trl_per_scratch_doubles(CHUNK) == CHUNK + 5 and L.trl_per_scratch_doubles(CHUNK + 1) == CHUNK + 11
    _rejects(L, L.trl_per_sample_rows(p, 0, p, p, p, 1, 0.4, p, p, p, None), "capacity 0 not in 1..16777216")
    _rejects(L, L.trl_per_sample_rows(p, (1 << 24) + 1, p, p, p, 1, 0.4, p, p, p, None), "not in 1..16777216")
    _rejects(L, L.trl_per_sample_rows(p, 8, p, p, p, 0, 0.4, p, p, p, None), "trl_per_sample_rows: empty batch")
    for k in range(7):
        args = [p] * 7
        args[k] = None
        prio, size, u, pos, idx, w, sc = args
        _rejects(L, L.trl_per_sample_rows(prio, 8, size, u, pos, 1, 0.4, idx, w, sc, None),
                 "trl_per_sample_rows: null pointer")
    _rejects(L, L.trl_twin_mse_loss_weighted(p, p, p, p, 0, p, p, p, p, p, p, None), "empty batch")
    _rejects(L, L.trl_twin_mse_loss_weighted(None, p, p, p, 8, p, p, p, p, p, p, None), "null pointer")
    _rejects(L, L.trl_twin_mse_loss_weighted(p, p, p, p, 8, p, None, p, p, p, p, None), "q2 given without g2")
    assert isinstance(buf, ctypes.Array)
