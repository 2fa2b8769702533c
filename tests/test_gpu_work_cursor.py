"""The hot window reduce hands its windows out through a work cursor: runs of consecutive windows while the ring is far from done,
single windows at the end, and the trailing partial window and the window that wraps the physical end of the ring in the same
launch.  These rings are large enough, and the grid small enough, that runs are handed out; the results must equal the C oracle's
on every window, reduce after reduce (the cursor is reset before each launch).  Run on an H100: pytest -m gpu."""
import numpy as np
import pytest

import synth

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("W", [1000, 1024])
def test_ring_cursor_runs_wrap_and_partial_windows(W):
    import gpud_b200 as g
    import mean_ema_ref as R
    F, cap = 64, 200_500
    first, second = 149_750, 200_500           # after the second push the ring has wrapped at an even start
    x = synth.gauge_stream(F, first + second, seed=W)
    thr = synth.thresholds_for(x)
    ctx = g.Context([0])
    r = g.Ring(ctx, F, cap, W, thresholds=thr)
    r.set_cta_reserve(100)                     # a smaller grid: most windows go out in runs
    for a, b in ((0, first), (first, first + second)):
        r.push(x[a:b])
        total, count, nw = r.counts()
        start = total % cap if total > cap else 0
        assert start % 2 == 0 and count % W != 0
        if total > cap:
            assert (cap - start) % W != 0          # one window wraps the physical end of the ring
        got = r.reduce_all()
        want = R.windows_fields(np.ascontiguousarray(x[total - count:total].T), W, thr)
        for k in ("min", "max", "p99"):
            assert np.array_equal(got[k].view(np.uint64), want[k].view(np.uint64)), (W, total, k)
        assert np.array_equal(got["n_over"].astype(np.uint64), want["n_over"].astype(np.uint64)), (W, total)
        R.check_mean_ema(got, want, what=(W, total))
    r.close()
    ctx.close()
