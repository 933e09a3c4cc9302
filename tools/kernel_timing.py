"""Quick device-resident timing of K1/K2 on schema S32 (development aid; bench.py is the contract)."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from k_llms_b200 import _native as K  # noqa: E402
from k_llms_b200 import synth  # noqa: E402


def timeit(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for a, b in evs:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    ts = sorted(a.elapsed_time(b) for a, b in evs)
    return ts[len(ts) // 2], ts[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=1_000_000)
    ap.add_argument("--n", type=int, nargs="+", default=[16])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--p-agree", type=float, default=0.8)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--interleave", action="store_true")
    ap.add_argument("--other", default="numeric", choices=["numeric", "read", "write", "copy", "none"])
    args = ap.parse_args()
    peak = 3350.0  # H100 SXM data sheet, GB/s; MEASURED_PEAKS.json overrides it
    try:
        peak = json.load(open(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")))["hbm_gbs"]
    except Exception:
        pass
    for n in args.n:
        N = args.records
        codes, none_code, vals = synth.s32_torch(N, n, 20260923, "cuda", p_agree=args.p_agree)
        c2, v2 = codes.view(N * 24, n), vals.view(N * 8, n)
        win = torch.empty(N * 24, dtype=torch.int32, device="cuda")
        t_v, t_v0 = timeit(lambda: K.vote(c2, none_code), args.iters, args.warmup)
        t_n, t_n0 = timeit(lambda: K.numeric(v2), args.iters, args.warmup)
        bv, bn = N * 24 * (4 * n + 8), N * 8 * (8 * n + 12)
        if args.interleave:  # as in bench.py: vote then numeric back to back, per-kernel events inside the loop
            big = torch.empty(128 * 1024 * 1024, dtype=torch.float64, device="cuda")  # 1 GiB
            other = {"numeric": lambda: K.numeric(v2), "read": lambda: big.sum(), "write": lambda: big[:12_000_000].zero_(),
                     "copy": lambda: big[:64 * 1024 * 1024].copy_(big[64 * 1024 * 1024:]), "none": lambda: None}[args.other]
            for _ in range(args.warmup):
                K.vote(c2, none_code); other()
            torch.cuda.synchronize()
            evs = [[torch.cuda.Event(enable_timing=True) for _ in range(3)] for _ in range(args.iters)]
            for e in evs:
                e[0].record(); K.vote(c2, none_code); e[1].record(); other(); e[2].record()
            torch.cuda.synchronize()
            tv = sorted(e[0].elapsed_time(e[1]) for e in evs)[len(evs) // 2]
            tn = sorted(e[1].elapsed_time(e[2]) for e in evs)[len(evs) // 2]
            print(json.dumps({"interleaved": args.other, "vote_ms": round(tv, 4), "numeric_ms": round(tn, 4), "vote_frac": round(bv / tv / 1e6 / peak, 3),
                              "numeric_frac": round(bn / tn / 1e6 / peak, 3)}), flush=True)
        out = {"n": n, "records": N, "p_agree": args.p_agree, "vote_ms": round(t_v, 4), "vote_GBps": round(bv / t_v / 1e6, 1), "vote_frac": round(bv / t_v / 1e6 / peak, 3),
               "numeric_ms": round(t_n, 4), "numeric_GBps": round(bn / t_n / 1e6, 1),
               "numeric_frac": round(bn / t_n / 1e6 / peak, 3),
               "records_per_s": round(N / ((t_v + t_n) / 1e3)), "both_frac": round((bv + bn) / (t_v + t_n) / 1e6 / peak, 3)}
        print(json.dumps(out), flush=True)
        del codes, vals


if __name__ == "__main__":
    main()
