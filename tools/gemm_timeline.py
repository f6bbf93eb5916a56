"""Phase timeline inside one launch of each step GEMM, fused and EPI_STORE (the in-kernel counterpart of gemm_bench.py).

  python tools/gemm_timeline.py --out DIR [--shapes ffn_up,to_q2.dX] [--width 2048]

Builds libb2d_trace.so (`make -C finetrainers_b200/csrc trace`: the GEMM compiled with -DB2D_GEMM_TRACE, a library of
its own; libb2d.so is untouched) and runs the twelve step shapes with gemm_bench.py's operands.  Each math warpgroup
stamps %globaltimer per tile: turn barrier entered / acquired, last MMA issued, MMAs drained, x tile arrived, end of each
epilogue pass, each TMA store issued and read; the producer adds the time it waited on empty stages.  Per shape and
epilogue (fused / store) the medians over the traced launch's tiles, in microseconds:

  main       turn acquired -> MMAs drained            issue    turn acquired -> last MMA issued
  turn       wait at the turn barrier                 x        MMAs drained -> x tile arrived (staged operand)
  pass1/2    epilogue pass (ends when every thread wrote the tile)
  rd1/rd2    TMA store issued -> store read (shared memory free again)
  epi        MMAs drained -> tile done (all passes, stores read)
  tail       per CTA: last MMA issued -> CTA exit     idle     per CTA: span minus the union of its main-loop windows
  prod       producer wait on empty stages per tile   span     first turn -> last exit of the launch

`idle` is time in which neither warpgroup of the CTA had a main loop in flight: the epilogue work the schedule did not
hide.  `main` under fused against store shows whether an epilogue slows the other warpgroup's concurrent main loop.
Results go to DIR/gemm_timeline.json and DIR/gemm_timeline.txt.  One run per session: %globaltimer ticks are tens of ns,
the medians are over hundreds of tiles.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from finetrainers_b200 import lib  # noqa: E402

SLOTS = 16
(TURN_WAIT, TURN, LAST_MMA, DRAINED, X, PASS1, ST1_ISSUE, ST1_READ, PASS2, ST2_ISSUE, ST2_READ, END, SM, MT, NT,
 KIND) = range(SLOTS)
MAX_TILES = 64
COLS = ["tiles", "main", "issue", "turn", "x", "pass1", "rd1", "pass2", "rd2", "epi", "tail", "idle", "prod", "span"]


def build_trace_lib(trace_dir):
    cmd = ["make", "-C", os.path.join(ROOT, "finetrainers_b200", "csrc"), "trace", f"TRACE_DIR={trace_dir}", "-j",
           str(min(8, os.cpu_count() or 1))]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise SystemExit("building libb2d_trace.so failed:\n" + r.stdout[-4000:] + r.stderr[-4000:])
    return os.path.join(trace_dir, "libb2d_trace.so")


def med(xs):
    xs = [x for x in xs if x is not None]
    return statistics.median(xs) / 1e3 if xs else None


def union_len(iv):
    tot, cur_s, cur_e = 0, None, None
    for s, e in sorted(iv):
        if cur_e is None or s > cur_e:
            if cur_e is not None:
                tot += cur_e - cur_s
            cur_s, cur_e = s, e
        else:
            cur_e = max(cur_e, e)
    return tot + (cur_e - cur_s if cur_e is not None else 0)


def analyse(rec):
    """rec: [ctas, MAX_TILES, 3, SLOTS] int64 -> medians of the phases (us) over tiles / CTAs"""
    col = {k: [] for k in COLS}
    t0, t1 = None, None
    for cta in range(rec.shape[0]):
        tiles = [rec[cta, t, r] for t in range(MAX_TILES - 1) for r in (0, 1) if rec[cta, t, r, KIND] == 1]
        exits = [rec[cta, MAX_TILES - 1, r, END] for r in (0, 1) if rec[cta, MAX_TILES - 1, r, KIND] == 2]
        if not tiles or not exits:
            continue
        col["tiles"].append(len(tiles) * 1e3)
        mains = []
        for x in tiles:
            def d(a, b):
                return int(x[b] - x[a]) if x[a] and x[b] else None
            col["main"].append(d(TURN, DRAINED))
            col["issue"].append(d(TURN, LAST_MMA))
            col["turn"].append(d(TURN_WAIT, TURN))
            col["x"].append(d(DRAINED, X))
            col["pass1"].append(d(X, PASS1))
            col["rd1"].append(d(ST1_ISSUE, ST1_READ))
            col["pass2"].append(d(ST1_READ, PASS2))
            col["rd2"].append(d(ST2_ISSUE, ST2_READ))
            col["epi"].append(d(DRAINED, END))
            mains.append((int(x[TURN]), int(x[DRAINED])))
        start, stop = min(int(x[TURN_WAIT]) for x in tiles), max(int(e) for e in exits)
        t0 = start if t0 is None else min(t0, start)
        t1 = stop if t1 is None else max(t1, stop)
        col["tail"].append(stop - max(int(x[LAST_MMA]) for x in tiles))
        col["idle"].append(stop - start - union_len(mains))
        for t in range(MAX_TILES - 1):
            p = rec[cta, t, 2]
            if p[KIND] == 1:
                col["prod"].append(int(p[TURN_WAIT]))
    out = {k: med(v) for k, v in col.items()}
    out["span"] = (t1 - t0) / 1e3 if t0 is not None else None
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for gemm_timeline.json / .txt")
    ap.add_argument("--trace-dir", default=os.path.join(ROOT, "finetrainers_b200", "csrc", "build", "trace"),
                    help="build directory of libb2d_trace.so")
    ap.add_argument("--shapes", default="", help="comma list of shape names (default: all twelve)")
    ap.add_argument("--width", type=int, default=2048)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    lib.LIB_PATH = build_trace_lib(os.path.abspath(args.trace_dir))  # before the first op loads the library
    import gemm_bench as GB
    GB.set_width(args.width)
    so = lib.load()
    so.b2d_gemm_trace_set.argtypes = [C.c_void_p, C.c_int]
    torch.manual_seed(0)
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    buf = torch.zeros(nsm * MAX_TILES * 3 * SLOTS, dtype=torch.int64, device="cuda")
    want = set(args.shapes.split(",")) if args.shapes else None
    rows, lines = [], []
    head = f"{'shape':<12} {'epi':<9} {'run':<5} " + " ".join(f"{c:>6}" for c in COLS)
    print(head)
    lines.append(head)
    for (name, N, K, b_mn, epi, K2, gn) in GB.SHAPES:
        if want and name not in want:
            continue
        sets = GB.make_sets(N, K, b_mn, epi, K2, gn)
        for fused in (True, False):
            run = GB.launcher(sets, N, K, b_mn, epi, K2, gn, fused, 0, 0)
            lib.check(so.b2d_gemm_trace_set(None, MAX_TILES), "gemm_trace_set")
            for i in range(3):
                run(i)
            torch.cuda.synchronize()
            buf.zero_()
            lib.check(so.b2d_gemm_trace_set(C.c_void_p(buf.data_ptr()), MAX_TILES), "gemm_trace_set")
            run(3)
            torch.cuda.synchronize()
            lib.check(so.b2d_gemm_trace_set(None, MAX_TILES), "gemm_trace_set")
            rec = buf.view(nsm, MAX_TILES, 3, SLOTS).cpu().numpy()
            r = analyse(rec)
            r.update(shape=name, epilogue=epi, run="fused" if fused else "store")
            rows.append(r)
            line = f"{name:<12} {epi:<9} {r['run']:<5} " + " ".join(
                f"{r[c]:>6.2f}" if r[c] is not None else f"{'-':>6}" for c in COLS)
            print(line, flush=True)
            lines.append(line)
        del sets
        torch.cuda.empty_cache()
    name = torch.cuda.get_device_name(0)
    foot = f"card: {name}; medians in us (tiles: per CTA)"
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        foot += f"; power limit, SM clock after the runs: {q}"
    except Exception:  # noqa: BLE001
        pass
    print(foot)
    lines.append(foot)
    with open(os.path.join(args.out, "gemm_timeline.json"), "w") as fh:
        json.dump({"card": name, "columns": COLS, "rows": rows}, fh, indent=1)
    with open(os.path.join(args.out, "gemm_timeline.txt"), "w") as fh:
        fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
