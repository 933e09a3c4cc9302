"""The list-alignment pre-pass on BASELINE config 3 records (nested JSON, depth 3, list fields; n = 8 by default), on one GPU:
  - records/s of align_json_batch (element similarities on the device, kc_alignsim.cuh) against per-record align_json spread
    over every host core (a process pool), both through the Python entry points, plus the native call kc_align_json_batch alone;
  - the share of element pairs the device pass decided;
  - the wall time of consolidate_json_packed on the same records as candidate texts, for this build and, with --parent-lib,
    for another build of the library (KLLMS_B200_LIB), the two alternated in fresh processes.
Prints one JSON line, with the GPU's name and power limit."""
import argparse
import ctypes
import json
import os
import random
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def config3(records, n, seed):
    from oracle.gen_golden import _record_candidates
    rng = random.Random(seed)
    return [json.loads(json.dumps(_record_candidates(rng, n, depth=3))) for _ in range(records)]


def _align_one(values):
    from k_llms_b200 import _native as K
    return K.align_json(values, 0.51)


def packed_times(records, n, seed, reps):
    """Wall times (ms) of consolidate_json_packed on config 3 texts, after one warm-up call."""
    from k_llms_b200 import _native as K
    texts = [[json.dumps(c) for c in rec] for rec in config3(records, n, seed)]
    blob, off, n = K.pack_texts(texts)
    K.consolidate_json_packed(blob, off, n).close()
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        res = K.consolidate_json_packed(blob, off, n)
        out.append((time.perf_counter() - t0) * 1e3)
        res.close()
    return out


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=20000)
    ap.add_argument("--n", type=int, default=8)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--seed", type=int, default=8)
    ap.add_argument("--parent-lib", default=None, help="another libkllms_b200.so to time consolidate_json_packed against")
    ap.add_argument("--packed-only", action="store_true", help=argparse.SUPPRESS)  # child process: one build's packed times
    args = ap.parse_args()
    if args.packed_only:
        from k_llms_b200 import _native as K
        have = ctypes.CDLL(K.LIB_PATH)  # an older build lacks the newer entry points: bind only what it has
        K._SIGNATURES = {k: v for k, v in K._SIGNATURES.items() if hasattr(have, k)}
        print(json.dumps(packed_times(args.records, args.n, args.seed, args.reps)))
        return
    import multiprocessing as mp
    import torch
    from k_llms_b200 import _native as K
    assert torch.cuda.is_available(), "align_throughput measures on a GPU"
    records = config3(args.records, args.n, args.seed)
    lib = K.load()

    # per-record align_json on every host core
    cores = os.cpu_count() or 1
    with mp.get_context("fork").Pool(cores) as pool:
        pool.map(_align_one, records[:cores * 4])  # warm-up: every worker loads the library
        host_s = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            expect = pool.map(_align_one, records, chunksize=max(1, len(records) // (cores * 8)))
            host_s.append(time.perf_counter() - t0)

    # align_json_batch through Python, and the native batch call alone
    K.align_json_batch(records[:200], device=0)
    batch_s, counts = [], {}
    for _ in range(args.reps):
        t0 = time.perf_counter()
        got = K.align_json_batch(records, device=0, counts=counts)
        batch_s.append(time.perf_counter() - t0)
    assert [json.dumps(g) for g in got] == [json.dumps(e) for e in expect], "align_json_batch differs from align_json"
    enc = [json.dumps(v).encode("ascii") for rec in records for v in rec]
    R, n = len(records), args.n
    texts = (ctypes.c_char_p * (R * n))(*enc)
    lens = (ctypes.c_int64 * (R * n))(*[len(b) for b in enc])
    native_s = []
    for _ in range(args.reps):
        out = (ctypes.c_void_p * (R * n))()
        status = (ctypes.c_int32 * R)()
        t0 = time.perf_counter()
        K.check(lib.kc_align_json_batch(ctypes.cast(texts, ctypes.c_void_p), ctypes.cast(lens, ctypes.c_void_p), R, n, 0.51, 0, 0,
                                        ctypes.cast(out, ctypes.c_void_p), ctypes.cast(status, ctypes.c_void_p), None))
        native_s.append(time.perf_counter() - t0)
        lib.kc_free_strings(ctypes.cast(out, ctypes.c_void_p), R * n)

    # consolidate_json_packed: this build and the parent build, alternated in fresh processes
    packed = {"this": [], "parent": []}
    for _ in range(2):
        for which in (["parent", "this"] if args.parent_lib else ["this"]):
            env = dict(os.environ)
            if which == "parent":
                env["KLLMS_B200_LIB"] = os.path.abspath(args.parent_lib)
            else:
                env.pop("KLLMS_B200_LIB", None)
            cmd = [sys.executable, os.path.abspath(__file__), "--packed-only", "--records", str(args.records), "--n", str(args.n),
                   "--seed", str(args.seed), "--reps", str(args.reps)]
            packed[which] += json.loads(subprocess.run(cmd, env=env, capture_output=True, text=True, check=True).stdout.strip().splitlines()[-1])

    med = statistics.median
    dp, hp = counts["device_pairs"], counts["host_pairs"]
    print(json.dumps({
        "gpu": gpu_info(), "records": R, "n": n, "host_cores": cores,
        "align_json_per_record_records_per_s": round(R / med(host_s)),
        "align_json_batch_records_per_s": round(R / med(batch_s)),
        "kc_align_json_batch_records_per_s": round(R / med(native_s)),
        "device_pairs": dp, "host_pairs": hp, "device_pair_share": round(dp / max(1, dp + hp), 4),
        "packed_wall_ms_this": round(med(packed["this"]), 2),
        "packed_wall_ms_parent": round(med(packed["parent"]), 2) if packed["parent"] else None,
        "packed_wall_ms_all": {k: [round(x, 2) for x in v] for k, v in packed.items()},
    }))


if __name__ == "__main__":
    main()
