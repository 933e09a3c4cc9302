"""BASELINE config 4 on the device: likelihood-weighted vote from per-token logprobs, n = 32, batch = 256K records.
K3 (kc_logprob_sum_f32: per-candidate fp32 sums of ragged token logprobs) then K3b (kc_weighted_vote_i32).  Prints one
JSON line with per-kernel times and HBM fractions (development aid; the semantics are self-defined, DESIGN.md section 5)."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from k_llms_b200 import _native as K  # noqa: E402


def timed(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for a, b in evs:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    return sorted(a.elapsed_time(b) for a, b in evs)[iters // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=262_144)
    ap.add_argument("--n", type=int, default=32)
    ap.add_argument("--fields", type=int, default=24)
    ap.add_argument("--min-tokens", type=int, default=32)
    ap.add_argument("--max-tokens", type=int, default=96)
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    peak = 3350.0  # H100 SXM data sheet, GB/s; MEASURED_PEAKS.json overrides it
    try:
        peak = json.load(open(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")))["hbm_gbs"]
    except Exception:
        pass
    R, n, F = args.records, args.n, args.fields
    g = torch.Generator(device="cuda").manual_seed(20260921 + 4)
    lens = torch.randint(args.min_tokens, args.max_tokens + 1, (R * n,), generator=g, device="cuda", dtype=torch.int64)
    offsets = torch.zeros(R * n + 1, dtype=torch.int64, device="cuda")
    torch.cumsum(lens, 0, out=offsets[1:])
    T = int(offsets[-1].item())
    lp = -torch.empty(T, dtype=torch.float32, device="cuda").exponential_(1.0, generator=g)
    truth = torch.randint(0, 6, (R, F, 1), generator=g, device="cuda", dtype=torch.int32)
    noise = torch.randint(0, 6, (R, F, n), generator=g, device="cuda", dtype=torch.int32)
    codes = torch.where(torch.rand((R, F, n), generator=g, device="cuda") < 0.8, truth.expand(-1, -1, n), noise).contiguous()
    sums = K.logprob_sum(lp, offsets)
    t_sum = timed(lambda: K.logprob_sum(lp, offsets), args.iters)
    seq = sums.view(R, n).contiguous()
    t_vote = timed(lambda: K.weighted_vote(codes, seq), args.iters)
    b_sum = T * 4 + (R * n + 1) * 8 + R * n * 4
    b_vote = R * F * n * 4 + R * n * 4 + R * F * 12
    print(json.dumps({"config": f"config 4: {R} records x {F} vote fields, n={n}, {args.min_tokens}-{args.max_tokens} tokens per candidate "
                                f"({T} token logprobs)",
                      "logprob_sum_ms": round(t_sum, 4), "logprob_sum_GBps": round(b_sum / t_sum / 1e6, 1),
                      "logprob_sum_frac": round(b_sum / t_sum / 1e6 / peak, 3),
                      "weighted_vote_ms": round(t_vote, 4), "weighted_vote_GBps": round(b_vote / t_vote / 1e6, 1),
                      "weighted_vote_frac": round(b_vote / t_vote / 1e6 / peak, 3),
                      "records_per_s": round(R / ((t_sum + t_vote) / 1e3)), "tokens_per_s": round(T / (t_sum / 1e3))}))


if __name__ == "__main__":
    main()
