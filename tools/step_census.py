"""Per-kernel census of one bench.py training step: per-kernel device time of one timed step, profiled with torch.profiler (CUDA
activities) in a run of its own, plus the live 128-row tiles of every SDF forward / train launch in that step (from the device counts).

    python tools/step_census.py [--workload 1080p-1M] [--step 5] [--json out.json]

bench.py itself runs (--steps 3 --warmup 3, no CPU / stock-CUDA legs); the profiler is switched on for one step only, between the
renderer's "step_begin" and "densify_stats" marks, with a device synchronise on both sides. The timing bench.py prints is discarded:
that step is not representative of an untraced one.
"""
import argparse
import collections
import contextlib
import io
import json
import os
import runpy
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "gs-sdf_b200")]

import torch  # noqa: E402

from gssdf_b200 import cabi, render  # noqa: E402


def live_tiles(n, n_variants, n_live, skip_base_variant, rows_per_tile):
    """tiles of a launch that do work, by the launch's own rules: sdf_fwd walks 128-row tiles of the [variant][point] layout and skips
    those beyond the live rows (and, with skip_base_variant, the variant-0 ones); sdf_train walks tiles of 128 / V whole points"""
    if rows_per_tile < 128:  # sdf_train with V variants per point
        return -(-n_live // rows_per_tile), -(-n // rows_per_tile)
    n_eval = n * max(n_variants, 1)
    n_tiles = -(-n_eval // 128)
    live = 0
    for t in range(n_tiles):
        base = 128 * t
        if base % n >= n_live and base % n + 128 <= n:
            continue
        if skip_base_variant and base + 128 <= n:
            continue
        live += 1
    return live, n_tiles


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="1080p-1M")
    ap.add_argument("--step", type=int, default=5, help="which call of the step (0-based, warm-up steps included) to profile")
    ap.add_argument("--json", help="also write the table as JSON here")
    args = ap.parse_args()

    state = dict(n=0, prof=None, launches=[])
    mark0 = render.SplatRenderer._mark

    def mark(self, name):
        mark0(self, name)
        if name == "step_begin":
            if state["n"] == args.step:
                torch.cuda.synchronize()
                state["prof"] = torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA])
                state["prof"].start()
            state["n"] += 1
        elif name == "densify_stats" and state["prof"] is not None and state["prof"] is not False:
            torch.cuda.synchronize()
            state["prof"].stop()
            state["result"], state["prof"] = state["prof"], False

    def record(kind, f):
        def g(net, x, *a, **kw):
            if state["prof"]:
                nl = kw.get("n_live")
                nv = kw.get("n_variants", 1) if kind == "sdf_fwd" else a[0]
                state["launches"].append(dict(kind=kind, n=int(x.shape[0]), n_variants=int(nv),
                                              skip_base_variant=bool(kw.get("skip_base_variant", False)),
                                              n_live=nl.clone() if nl is not None else None))
            return f(net, x, *a, **kw)
        return g

    render.SplatRenderer._mark = mark
    for name in ("sdf_fwd", "sdf_train"):
        wrapped = record(name, getattr(cabi, name))
        setattr(cabi, name, wrapped)
        setattr(render.cabi, name, wrapped)
    sys.argv = ["bench.py", "--gpus", "1", "--steps", "3", "--warmup", "3", "--workload", args.workload, "--no-cpu-baseline", "--no-stock-cuda"]
    with contextlib.redirect_stdout(io.StringIO()):
        try:
            runpy.run_path(os.path.join(ROOT, "bench.py"), run_name="__main__")
        except SystemExit:
            pass
    assert "result" in state, f"step {args.step} was never profiled ({state['n']} steps ran)"

    per = collections.OrderedDict()
    for e in state["result"].events():
        if e.device_type == torch.autograd.DeviceType.CUDA and e.device_time > 0:
            k = e.name.split("(")[0]
            if k.startswith("void "):
                k = k[5:]
            per.setdefault(k, []).append(e.device_time)
    rows = sorted(((sum(v), len(v), k) for k, v in per.items()), reverse=True)
    total = sum(r[0] for r in rows)
    name = torch.cuda.get_device_name()
    print(f"# {name}, one {args.workload} step (call {args.step}), kernel device time")
    for us, n, k in rows:
        print(f"{us:9.1f} us {100 * us / total:5.1f}%  x{n:<3d} {k[:100]}")
    print(f"{total:9.1f} us  sum over kernels (the two streams overlap; this is not the step time)")
    tiles = []
    print("# SDF launches of that step: live 128-row tiles / tiles of the capacity layout")
    for L in state["launches"]:
        nl = int(L["n_live"][0]) if L["n_live"] is not None else L["n"]
        nl = min(nl, L["n"])
        rpt = 128 if L["kind"] == "sdf_fwd" else 128 // L["n_variants"]
        live, cap = live_tiles(L["n"], L["n_variants"], nl, L["skip_base_variant"], rpt)
        tiles.append(dict(L, n_live=nl, live_tiles=live, tiles=cap))
        print(f"  {L['kind']:9s} n={L['n']:<8d} n_live={nl:<8d} V={L['n_variants']} skip_base={int(L['skip_base_variant'])}  "
              f"live tiles {live} of {cap}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(device=name, kernels=[dict(name=k, us=us, launches=n) for us, n, k in rows], sdf_launches=tiles), f, indent=1)


if __name__ == "__main__":
    main()
