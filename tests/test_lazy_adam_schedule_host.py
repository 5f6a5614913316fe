"""Host restatement of the lazy SH Adam schedule (render.GsSdfTrainer.adam_all + the SH forward's catch-up): which steps sweep, the ring
slots the replays read, and that no row ever falls a window behind over a long random visibility trace."""
import numpy as np
import pytest

pytest.importorskip("torch")


def test_window_matches_header():
    from gssdf_b200 import _lib, cabi
    src = open(_lib.HEADER).read()
    assert f"#define GSSDF_ADAM_WINDOW {cabi.ADAM_WINDOW}" in src
    assert cabi.ADAM_WINDOW & (cabi.ADAM_WINDOW - 1) == 0  # the kernels take s % WINDOW as s & (WINDOW - 1)
    fields = dict(_lib.STRUCTS["gssdf_adam_replay"]._fields_)
    assert fields["inv_sqrt_bc2"]._length_ == cabi.ADAM_WINDOW and fields["step_size"]._length_ == 2 * cabi.ADAM_WINDOW


def test_sweep_steps():
    from gssdf_b200 import cabi, render
    W = cabi.ADAM_WINDOW
    assert [t for t in range(1, 3 * W + 1) if render.sh_sweep_step(t)] == [W, 2 * W, 3 * W]


@pytest.mark.parametrize("p_visible", [0.0, 0.02, 0.15, 0.9])
def test_rows_stay_within_the_window(p_visible):
    """Every replay reads the slots of steps last+1 .. to, all within the WINDOW steps that end at the current step (the ring then
    still holds them: slot s % WINDOW is overwritten only by step s + WINDOW)."""
    from gssdf_b200 import cabi, render
    W = cabi.ADAM_WINDOW
    rng = np.random.default_rng(int(p_visible * 100))
    n_rows, steps = 500, 20 * W + 17
    last = np.zeros(n_rows, np.int64)
    newest = 0  # newest step whose scalars were pushed

    def replay(rows, to):
        for r in rows:
            span = list(range(last[r] + 1, to + 1))
            assert len(span) <= W - 1, (r, last[r], to)
            assert all(newest - W < s <= newest for s in span)
            assert len({s % W for s in span}) == len(span)

    for t in range(1, steps + 1):
        vis = np.flatnonzero(rng.random(n_rows) < p_visible)
        replay(vis, t - 1)  # catch-up in the SH forward of step t (the trainer has pushed step t - 1)
        last[vis] = t - 1
        newest = t  # adam_all pushes step t, then updates
        rows = np.arange(n_rows) if render.sh_sweep_step(t) else vis
        replay(rows, t - 1)
        last[rows] = t
        assert (t - last).max() <= W - 1 or render.sh_sweep_step(t)
    replay(np.arange(n_rows), steps)  # the flush of a parameter read
