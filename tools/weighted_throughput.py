"""K3b over ragged records (kc_weighted_vote_groups_i8) against K1 on the same int8 cells (kc_vote_i8): 24 vote fields per
record (S32's vote fields), 1 M records at n = 16 and 256 K at n = 32 (BASELINE config 4's size).  Weighted and unweighted
launches are timed alternately, twice each; prints one JSON line per shape with the GPU name and power limit read in the same
run.  Then the device JSON path end to end, weighted (kc_consolidate_json_packed_weighted, seeded sums) against count votes,
alternated twice on 1 M S32 texts at n = 16, with the kc_json_stats stage split (development aid; the weighting is
self-defined, DESIGN.md section 5)."""
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from k_llms_b200 import _native as K  # noqa: E402
from tools.config4_timing import timed  # noqa: E402

PEAK_GBS = 3350.0  # H100 SXM data sheet


def gpu_card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        out = ""
    return out or torch.cuda.get_device_name()


def main():
    card = gpu_card()
    F = 24
    for R, n in ((1_048_576, 16), (262_144, 32)):
        g = torch.Generator(device="cuda").manual_seed(20261016 + n)
        G = R * F
        truth = torch.randint(0, 6, (G, 1), generator=g, device="cuda", dtype=torch.int8)
        noise = torch.randint(-1, 6, (G, n), generator=g, device="cuda", dtype=torch.int8)
        codes = torch.where(torch.rand((G, n), generator=g, device="cuda") < 0.8, truth.expand(-1, n), noise).contiguous()
        # records in shuffled order, as the device JSON path reserves them
        rec = torch.randperm(R, generator=g, device="cuda").to(torch.int32).repeat_interleave(F)
        seq = -torch.empty((R, n), dtype=torch.float32, device="cuda").exponential_(8.0, generator=g)
        times = {"weighted": [], "unweighted": []}
        for _ in range(2):
            times["weighted"].append(timed(lambda: K.weighted_vote_groups(codes, rec, seq), 10))
            times["unweighted"].append(timed(lambda: K.vote_i8(codes), 10))
        b_w = G * n + G * 4 + R * n * 4 + G * 12  # cells, record index, sums, results
        b_u = G * n + G * 8
        tw, tu = min(times["weighted"]), min(times["unweighted"])
        print(json.dumps({"gpu": card, "shape": f"{R} records x {F} vote fields, n={n}",
                          "weighted_ms": [round(t, 4) for t in times["weighted"]],
                          "unweighted_ms": [round(t, 4) for t in times["unweighted"]],
                          "weighted_GBps": round(b_w / tw / 1e6, 1), "weighted_frac_of_3.35TBps": round(b_w / tw / 1e6 / PEAK_GBS, 3),
                          "unweighted_GBps": round(b_u / tu / 1e6, 1), "unweighted_frac_of_3.35TBps": round(b_u / tu / 1e6 / PEAK_GBS, 3),
                          "weighted_over_unweighted": round(tw / tu, 2)}))
    # end to end on the device JSON path: 1 M S32 records of n = 16 candidate texts, weighted (seeded sums) against count votes
    import numpy as np
    R, n = 1_000_000, 16
    blob, off = K.s32_texts_packed(R, n, 20261016)
    seq = (-np.random.default_rng(5).exponential(8.0, R * n)).astype(np.float32)
    runs = {"weighted": [], "unweighted": []}
    for _ in range(2):
        for kind in ("weighted", "unweighted"):
            res = (K.consolidate_json_packed_weighted(blob, off, n, seq) if kind == "weighted"
                   else K.consolidate_json_packed(blob, off, n))
            st = res.stats.as_dict()
            res.close()
            runs[kind].append({k: (round(v, 3) if isinstance(v, float) else v) for k, v in st.items()
                               if k in ("wall_ms", "h2d_ms", "plan_ms", "kernel_ms", "emit_ms", "d2h_ms", "n_device", "n_host", "n_python")})
    print(json.dumps({"gpu": card, "shape": f"end to end, kc_consolidate_json_packed(_weighted), {R} S32 records, n={n}",
                      "weighted": runs["weighted"], "unweighted": runs["unweighted"],
                      "weighted_records_per_s": round(R / (min(r["wall_ms"] for r in runs["weighted"]) / 1e3)),
                      "unweighted_records_per_s": round(R / (min(r["wall_ms"] for r in runs["unweighted"]) / 1e3))}))


if __name__ == "__main__":
    main()
