"""The async entry points on the device (KC_JSON_NUMERIC_MEDOID) against the Python async route, and K5 against K2.

1. requests/s and p50 / p99 latency of async_consolidate_parsed_chat_completions at 1, 16 and 256 concurrent requests on one event
   loop, on S32 texts (SURVEY.md section 8d) or (--workload invoice_optional) invoice texts whose candidates reorder, drop and add
   keys, (invoice_lines) invoice texts whose `items` is a list of line items, or (mixed_lines) S32 and invoice_lines requests
   interleaved, or (unicode_invoice) invoice texts with accented, curly-quoted free text (tools/jsonpacked_throughput.py), at n = 3 and 16: the native route (device JSON path, requests combined per
   device call) against the Python async route (_consensus_async) on the same contents.
2. kernel time of K5 (kc_numeric_medoid_f64) against K2 (kc_numeric_f64) on the same S32 numeric cells, 1 M records x 8 fields,
   at n = 4, 16, 32, 64 (CUDA events, median of 20 launches).
Prints one JSON line per row, with the GPU name and power limit read in the same run."""
import asyncio
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from k_llms_b200 import _native as K  # noqa: E402
from k_llms_b200 import synth  # noqa: E402
from k_llms_b200.utils import consolidation as C  # noqa: E402
from tools.config4_timing import timed  # noqa: E402
from tools.weighted_throughput import gpu_card  # noqa: E402


async def _no_embeddings(texts):
    raise RuntimeError("no embeddings service in this measurement")


def s32_completions(count, n, seed, workload="s32"):
    from openai.types.chat import ParsedChatCompletion
    def s32(count):
        blob, off = K.s32_texts_packed(count, n, seed, pinned=False)
        raw = bytes(blob[:int(off[-1])])
        return [[raw[off[r * n + c]:off[r * n + c + 1]].decode("ascii") for c in range(n)] for r in range(count)]
    if workload == "invoice_optional":
        from tools.jsonpacked_throughput import invoice_texts
        records = invoice_texts(count, n, seed, optional=True)
    elif workload == "invoice_lines":
        from tools.jsonpacked_throughput import invoice_lines_texts
        records = invoice_lines_texts(count, n, seed)
    elif workload == "unicode_invoice":
        from tools.jsonpacked_throughput import invoice_texts
        records = invoice_texts(count, n, seed, accents=True)
    elif workload == "mixed_lines":
        from tools.jsonpacked_throughput import invoice_lines_texts
        records = [r for pair in zip(s32(count // 2), invoice_lines_texts(count - count // 2, n, seed)) for r in pair]
    else:
        records = s32(count)
    out = []
    for texts in records:
        out.append(ParsedChatCompletion.model_validate({
            "id": "x", "object": "chat.completion", "created": 0, "model": "m",
            "choices": [{"index": i, "finish_reason": "stop", "message": {"role": "assistant", "content": t}} for i, t in enumerate(texts)]}))
    return out


async def _run(completions, concurrency):
    """Every completion once, `concurrency` requests in flight; returns (wall seconds, per-request latencies)."""
    lat = []
    it = iter(completions)

    async def worker():
        for comp in it:
            t0 = time.perf_counter()
            await C.async_consolidate_parsed_chat_completions(comp, _no_embeddings, None)
            lat.append(time.perf_counter() - t0)
    t0 = time.perf_counter()
    await asyncio.gather(*(worker() for _ in range(concurrency)))
    return time.perf_counter() - t0, lat


def requests_rows(card, workload="s32", count=2048):
    native_route = C._consensus_of_choices_native_async

    async def python_only(*a, **k):
        return None
    for n in (3, 16):
        comps = s32_completions(count, n, 20261016 + n, workload)
        for conc in (1, 16, 256):
            row = {"what": "async_requests", "workload": workload, "n": n, "concurrency": conc, "gpu": card}
            for route in ("python", "native", "python", "native"):  # alternated twice; the faster run of each is reported
                C._consensus_of_choices_native_async = native_route if route == "native" else python_only
                k = len(comps) if route == "native" else min(256, len(comps))
                asyncio.run(_run(comps[:64], min(conc, 64)))  # warm-up
                wall, lat = asyncio.run(_run(comps[:k], conc))
                rps = k / wall
                if rps > row.get(f"{route}_req_per_s", 0.0):
                    row[f"{route}_req_per_s"] = round(rps, 1)
                    row[f"{route}_p50_ms"] = round(float(np.percentile(lat, 50)) * 1e3, 3)
                    row[f"{route}_p99_ms"] = round(float(np.percentile(lat, 99)) * 1e3, 3)
            C._consensus_of_choices_native_async = native_route
            print(json.dumps(row), flush=True)


def kernel_rows(card):
    R, F = 1 << 20, 8
    for n in (4, 16, 32, 64):
        block = 1 << 16  # S32 numeric cells of 64 K records, tiled to 1 M records
        _, _, vals = synth.s32_numpy(block, n, 20261016 + n)
        cells = torch.from_numpy(np.ascontiguousarray(vals.reshape(-1, n))).cuda().repeat(R // block, 1).contiguous()
        G = cells.shape[0]
        assert G == R * F
        best = torch.empty(G, dtype=torch.int32, device="cuda")
        avg = torch.empty(G, dtype=torch.float64, device="cuda")
        value = torch.empty(G, dtype=torch.float64, device="cuda")
        meta = torch.empty(G, dtype=torch.int32, device="cuda")
        sp = torch.cuda.current_stream().cuda_stream
        lib = K.load()
        k5 = lambda: K.check(lib.kc_numeric_medoid_f64(cells.data_ptr(), G, n, best.data_ptr(), avg.data_ptr(), sp))  # noqa: E731
        k2 = lambda: K.check(lib.kc_numeric_f64(cells.data_ptr(), G, n, 0.03, 1e-6, value.data_ptr(), meta.data_ptr(), sp))  # noqa: E731
        t5 = min(timed(k5, 20), timed(k5, 20))
        t2 = min(timed(k2, 20), timed(k2, 20))
        print(json.dumps({"what": "kernel", "records": R, "fields": F, "n": n, "k5_ms": round(t5, 3), "k2_ms": round(t2, 3),
                          "k5_over_k2": round(t5 / t2, 2), "gpu": card}), flush=True)
        del cells, best, avg, value, meta
        torch.cuda.empty_cache()


def main():
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", choices=["s32", "invoice_optional", "invoice_lines", "mixed_lines", "unicode_invoice"], default="s32",
                    help="the request rows' candidate texts")
    ap.add_argument("--requests", type=int, default=2048, help="requests per row (the Python route runs at most 256 of them)")
    ap.add_argument("--requests-only", action="store_true", help="skip the K5 / K2 kernel rows")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    card = gpu_card()
    if not args.requests_only:
        kernel_rows(card)
    requests_rows(card, args.workload, args.requests)


if __name__ == "__main__":
    main()
