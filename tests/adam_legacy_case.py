"""A fixed sequence of gssdf_adam_step calls over dense, half-shadow and lazy row groups, 70 steps across a GSSDF_ADAM_WINDOW boundary.
tests/golden/adam_legacy.npz holds its inputs and the outputs the single-clock optimiser produced before the per-group clocks entry was
added; test_gpu_gs_train.py replays it and compares bit for bit."""
import numpy as np
import torch

from gssdf_b200 import cabi
from gssdf_b200.render import sh_sweep_step

STEPS = 70
N_DENSE, N_HALF, HALF_OFF, ROWS, W0, W1 = 1000, 1027, 1002, 200, 3, 9
ROW_OFF = HALF_OFF + N_HALF + 1  # odd offset: the row groups and the half group take the scalar path of the dense kernel
N_TOTAL = ROW_OFF + ROWS * (W0 + W1)


def make_inputs(seed=0):
    rng = np.random.default_rng(seed)
    f = lambda *s: rng.standard_normal(s).astype(np.float32)
    # four visit lists of 60, 80, 100 and 120 distinct rows, padded with -1 to one width
    ids = np.stack([np.pad(rng.permutation(ROWS)[:60 + 20 * k], (0, 60 - 20 * k), constant_values=-1) for k in range(4)])
    return dict(p0=f(N_TOTAL), grads=f(4, N_TOTAL) * np.float32(0.01), row_ids=ids.astype(np.int64))


def groups(lr_scale=1.0):
    return [(0, N_DENSE, 1e-3 * lr_scale, False, 0), (HALF_OFF, N_HALF, 5e-3 * lr_scale, True, 0),
            (ROW_OFF, ROWS * W0, 2.5e-3 * lr_scale, False, W0), (ROW_OFF + ROWS * W0, ROWS * W1, 1.25e-4 * lr_scale, False, W1)]


def run(inp, dev, step_fn=None):
    """Runs the sequence; step_fn(p, g, m, v, groups, t, **kw) defaults to cabi.adam_step. Returns params, exp_avg, exp_avg_sq, half."""
    step_fn = step_fn or cabi.adam_step
    t_ = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    p, m, v = t_(inp["p0"]), torch.zeros(N_TOTAL, device=dev), torch.zeros(N_TOTAL, device=dev)
    g = torch.zeros(N_TOTAL, device=dev)
    half = torch.zeros(N_HALF, dtype=torch.float16, device=dev)
    last = torch.zeros(ROWS, dtype=torch.int32, device=dev)
    replay = cabi.AdamReplay(last)
    counts = torch.zeros(cabi.COUNTS_INTS, dtype=torch.int32, device=dev)
    grads, ids_all = t_(inp["grads"]), inp["row_ids"]
    for t in range(1, STEPS + 1):
        k = t % 4
        ids_np = ids_all[k][ids_all[k] >= 0]
        ids = t_(ids_np)
        g.copy_(grads[k])
        rows = torch.zeros(ROWS, device=dev)
        rows[ids] = 1.0
        g[ROW_OFF:ROW_OFF + ROWS * W0].view(ROWS, W0).mul_(rows[:, None])
        g[ROW_OFF + ROWS * W0:].view(ROWS, W1).mul_(rows[:, None])
        grp = groups(1.0 + 0.01 * t)
        replay.push(t, grp[2][2], grp[3][2])
        counts[0] = len(ids_np)
        row = {} if sh_sweep_step(t) else dict(row_ids=ids, row_count=counts, row_cap=len(ids_np))
        step_fn(p, g, m, v, grp, t, grad_scale=0.5 if t % 3 == 0 else 1.0, zero_grads=True, table_half=half, replay=replay, **row)
    step_fn(p, g, m, v, groups(1.0 + 0.01 * STEPS)[2:], STEPS, replay=replay, replay_only=True)
    return dict(params=p.cpu().numpy(), exp_avg=m.cpu().numpy(), exp_avg_sq=v.cpu().numpy(), half=half.cpu().numpy())
