"""Times every large GEMM of the training step at its real shape, layout and epilogue (M = 2688: one 49x512x768 sample).

  python tools/gemm_bench.py [--iters 30] [--block-n 0,128,192,256] [--cta-pair 0,2] [--width 2048] [--json OUT]

Per shape and tile choice: the fused launch as the step issues it, the same launch with EPI_STORE (no bias, gate, residual
or second output; the LoRA extension stays, it is part of the contraction), and torch.mm on the same bf16 main operands
(cuBLAS, no epilogue, no extension) as the practical ceiling of the card.  CUDA events over `--iters` back-to-back
launches after a warm-up; every launch reads and writes the next of several operand sets (> 50 MB together), so L2 does
not hold the previous launch's data.  TFLOP/s counts 2 M N (K + K2).  The card name, power limit and the median SM clock
over the timed loops are printed beside the table.
"""
import argparse
import json
import math
import os
import statistics
import sys
import threading
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from finetrainers_b200 import ops  # noqa: E402

M, D, RP = 2688, 2048, 64
ROTATE_BYTES = 64 << 20

def shapes(D):
    """name, N, K, dX (MN-major B), epilogue, K2 (LoRA extension), a2_group_n of the twelve step GEMMs at width D"""
    return [
        ("qkv", 3 * D, D, False, "store", RP, D),
        ("to_out", D, D, False, "gate_res", RP, 0),
        ("to_q2", D, D, False, "store", RP, 0),
        ("to_out2", D, D, False, "res", RP, 0),
        ("ffn_up", 4 * D, D, False, "gelu2", 0, 0),
        ("ffn_down", D, 4 * D, False, "gate_res", 0, 0),
        ("qkv.dX", D, 3 * D, True, "store", 3 * RP, 0),
        ("to_out.dX", D, D, True, "store", RP, 0),
        ("to_q2.dX", D, D, True, "res_gate2", RP, 0),
        ("to_out2.dX", D, D, True, "store", RP, 0),
        ("ffn_down.dX", 4 * D, D, True, "dgelu", 0, 0),
        ("ffn_up.dX", D, 4 * D, True, "store", 0, 0),
    ]


def set_width(width):
    """The residual width the shapes, gate tables and temb stride are built for (2048: LTX-2B, 4096: LTX-13B)."""
    global D, SHAPES
    D, SHAPES = width, shapes(width)


SHAPES = shapes(D)


class Clock:
    """Median SM clock sampled in-process through NVML every 50 ms while `on` is set."""

    def __init__(self):
        self.on, self.stop, self.mhz, self.h = False, False, [], None
        self.name, self.power_w = torch.cuda.get_device_name(0), None
        try:
            import pynvml as nv
            nv.nvmlInit()
            vis = os.environ.get("CUDA_VISIBLE_DEVICES", "").split(",")[0].strip()
            self.h = nv.nvmlDeviceGetHandleByIndex(int(vis) if vis.isdigit() else 0)
            self.power_w = nv.nvmlDeviceGetPowerManagementLimit(self.h) / 1000.0
            self.nv = nv
            self.t = threading.Thread(target=self._run, daemon=True)
            self.t.start()
        except Exception as e:  # noqa: BLE001
            self.err = repr(e)

    def _run(self):
        while not self.stop:
            if self.on:
                try:
                    self.mhz.append(self.nv.nvmlDeviceGetClockInfo(self.h, self.nv.NVML_CLOCK_SM))
                except Exception:  # noqa: BLE001
                    pass
            time.sleep(0.05)

    def finish(self):
        self.stop = True
        if self.h is not None:
            self.t.join(timeout=2)
        return statistics.median(self.mhz) if self.mhz else None


def rnd(*shape, scale=1.0):
    return (torch.randn(*shape, device="cuda") * scale).bfloat16()


def make_sets(N, K, b_mn, epi, K2, a2_group_n):
    """Operand sets for one shape: enough of them that consecutive launches touch > ROTATE_BYTES of distinct memory."""
    def one():
        s = {"A": rnd(M, K), "B": rnd(K, N, scale=0.02) if b_mn else rnd(N, K, scale=0.02),
             "out": torch.empty(M, N, device="cuda", dtype=torch.bfloat16)}
        if K2:
            s["A2"] = rnd(M, K2 * (N // a2_group_n) if a2_group_n else K2, scale=0.3)
            s["B2"] = rnd(K2, N, scale=0.02) if b_mn else rnd(N, K2, scale=0.02)
        if not b_mn:
            s["bias"] = rnd(N, scale=0.1)
        if epi in ("gate_res", "res", "res_gate2"):
            s["res"] = rnd(M, N)
        if epi == "dgelu":
            s["aux"] = rnd(M, N)
        if epi in ("gelu2", "res_gate2"):
            s["out2"] = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
        if epi in ("gate_res", "res_gate2"):
            s["gtab"], s["gtemb"] = rnd(N, scale=0.1), rnd(1, 6 * D, scale=0.1)
        return s
    first = one()
    per = sum(t.numel() * t.element_size() for t in first.values())
    return [first] + [one() for _ in range(max(2, math.ceil(ROTATE_BYTES / per)) - 1)]


def launcher(sets, N, K, b_mn, epi, K2, a2_group_n, fused, block_n, cta_pair):
    def run(i):
        s = sets[i % len(sets)]
        kw = dict(M=M, N=N, K=K, b_mn=b_mn, block_n=block_n, cta_pair=cta_pair)
        if K2:
            kw.update(A2=s["A2"], B2=s["B2"], K2=K2, a2_group_n=a2_group_n)
        if fused:
            kw["bias"] = s.get("bias")
            if epi == "gelu2":
                kw.update(epi=ops.EPI_GELU, out2=s["out2"])
            elif epi == "gate_res":
                kw.update(epi=ops.EPI_GATE_RES, res=s["res"], gate_table=s["gtab"], gate_temb=s["gtemb"],
                          temb_stride=6 * D, rows_per_sample=M)
            elif epi == "res":
                kw.update(epi=ops.EPI_GATE_RES, res=s["res"])
            elif epi == "res_gate2":
                kw.update(epi=ops.EPI_GATE_RES, res=s["res"], gate2_table=s["gtab"], gate2_temb=s["gtemb"],
                          out2=s["out2"], temb_stride=6 * D, rows_per_sample=M)
            elif epi == "dgelu":
                kw.update(epi=ops.EPI_MUL_DGELU, aux=s["aux"])
        ops.gemm(s["A"], s["B"], s["out"], **kw)
    return run


def cublas(sets, b_mn):
    def run(i):
        s = sets[i % len(sets)]
        torch.mm(s["A"], s["B"] if b_mn else s["B"].t(), out=s["out"])
    return run


def time_ms(fn, iters, clock):
    for i in range(3):
        fn(i)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    clock.on = True
    e0.record()
    for i in range(iters):
        fn(i)
    e1.record()
    torch.cuda.synchronize()
    clock.on = False
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--block-n", default="0", help="comma list of tile widths (0 = the library's automatic choice)")
    ap.add_argument("--cta-pair", default="0", help="comma list of cta_pair values (0 auto, 1 single CTA, 2 pairs)")
    ap.add_argument("--shapes", default="", help="comma list of shape names (default: all twelve)")
    ap.add_argument("--no-cublas", action="store_true")
    ap.add_argument("--width", type=int, default=D, help="residual width D of the shapes (4096: the 13B geometry)")
    ap.add_argument("--json", default=None, help="also write the rows as JSON to this path")
    args = ap.parse_args()
    if args.iters < 30:
        raise SystemExit("--iters must be >= 30")
    set_width(args.width)
    torch.manual_seed(0)
    clock = Clock()
    bns = [int(x) for x in args.block_n.split(",")]
    pairs = [int(x) for x in args.cta_pair.split(",")]
    want = set(args.shapes.split(",")) if args.shapes else None
    rows = []
    print(f"{'shape':<12} {'N':>5} {'K':>5} {'K2':>4} {'epi':<9} {'bn':>3} {'pair':>4} {'fused us':>9} {'TF/s':>6} "
          f"{'store us':>9} {'epi us':>7} {'cuBLAS us':>9} {'TF/s':>6}")
    tot = {"fused": 0.0, "store": 0.0, "cublas": 0.0}
    for (name, N, K, b_mn, epi, K2, gn) in SHAPES:
        if want and name not in want:
            continue
        sets = make_sets(N, K, b_mn, epi, K2, gn)
        flop = 2.0 * M * N * (K + K2)
        cb = None if args.no_cublas else time_ms(cublas(sets, b_mn), args.iters, clock)
        for bn in bns:
            for cp in pairs:
                try:
                    f = time_ms(launcher(sets, N, K, b_mn, epi, K2, gn, True, bn, cp), args.iters, clock)
                    s = time_ms(launcher(sets, N, K, b_mn, epi, K2, gn, False, bn, cp), args.iters, clock)
                except Exception as e:  # noqa: BLE001  (a tile choice the library rejects for this shape)
                    print(f"{name:<12} bn={bn} pair={cp}: {str(e).splitlines()[0]}")
                    continue
                row = {"shape": name, "N": N, "K": K, "K2": K2, "epi": epi, "block_n": bn, "cta_pair": cp,
                       "fused_us": f * 1e3, "fused_tflops": flop / f / 1e9, "store_us": s * 1e3,
                       "epilogue_us": (f - s) * 1e3,
                       "cublas_us": cb * 1e3 if cb else None,
                       "cublas_tflops": 2.0 * M * N * K / cb / 1e9 if cb else None}
                rows.append(row)
                if bn == bns[0] and cp == pairs[0]:
                    tot["fused"] += f
                    tot["store"] += s
                    tot["cublas"] += cb or 0.0
                print(f"{name:<12} {N:>5} {K:>5} {K2:>4} {epi:<9} {bn:>3} {cp:>4} {f * 1e3:>9.1f} {flop / f / 1e9:>6.0f} "
                      f"{s * 1e3:>9.1f} {(f - s) * 1e3:>7.1f} "
                      + (f"{cb * 1e3:>9.1f} {2.0 * M * N * K / cb / 1e9:>6.0f}" if cb else ""), flush=True)
        del sets
        torch.cuda.empty_cache()
    mhz = clock.finish()
    print(f"sum over shapes (first tile choice): fused {tot['fused']:.3f} ms, store {tot['store']:.3f} ms, "
          f"cuBLAS {tot['cublas']:.3f} ms; x28 blocks: fused {28 * tot['fused']:.1f} ms")
    print(f"card: {clock.name}, power limit {clock.power_w} W, median SM clock {mhz} MHz")
    if args.json:
        with open(args.json, "w") as fh:
            json.dump({"card": clock.name, "power_limit_w": clock.power_w, "sm_mhz_median": mhz, "rows": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
