"""Throughput of H1g (kc_consolidate_json_packed): S32 candidate texts in pinned host memory -> consensus / likelihoods texts,
wall clock around the C-ABI call, with the per-stage device times the call reports.  One JSON line per configuration."""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from k_llms_b200 import _native as K  # noqa: E402


# the optional-keys workloads: each candidate independently reorders its keys (at every level), drops one, adds an extra one,
# and (nested) sets a sub-object to None or leaves it out, with these probabilities
P_REORDER, P_DROP, P_EXTRA, P_NULL_SUB, P_MISSING_SUB = 0.5, 0.2, 0.2, 0.1, 0.05


def invoice_texts(records, n, seed, nested=False, optional=False, accents=False):
    """An extraction-like schema with FREE-TEXT fields (multi-word strings -> similarity medoid, K4) next to enums, bools and
    numbers: 4 phrases, 3 enums, 2 bools, 3 numbers per record; every candidate copies the record's truth with probability 0.8
    per field, otherwise a variant (case / punctuation / one word changed / another value), None with probability 0.05.
    optional: the candidates differ in shape as well (P_* above): the device path's key-union round.  accents: the free-text
    fields hold accented letters, curly quotes, dashes and the euro sign, as raw UTF-8 (the enums stay ASCII): the device
    path's KC_JSON_UNICODE medoids."""
    import random
    rng = random.Random(seed)
    vendors = ["Acme Industrial Supply Co", "Globex Logistics and Freight", "Initech Software Services Ltd", "Umbrella Medical Devices Inc"]
    streets = ["12 Rue de la Paix 75002 Paris", "221B Baker Street London NW1", "1600 Amphitheatre Parkway Mountain View", "5 Avenue Anatole France Paris"]
    terms = ["net 30 days from invoice date", "payment due on receipt", "2 percent 10 net 30", "net 60 days end of month"]
    notes = ["deliver to the rear loading dock", "fragile handle with care", "partial shipment remaining items to follow", "customer will collect in person"]
    if accents:
        vendors = ["Société Générale d’Équipement", "Müller & Söhne Großhandel GmbH", "Café “Le Pâtissier” Fournitures", "Łódź Ćwiczenia Spółka z o.o."]
        streets = ["12 Rue de la Paix — 75002 Paris", "Königstraße 5, 70173 Stuttgart", "Praça da Sé 108 — São Paulo", "Calle de Alcalá 48, Madrid"]
        terms = ["net 30 days — 2 % escompte", "payment due on receipt (€)", "Zahlung binnen 14 Tagen netto", "net 60 days “end of month”"]
        notes = ["livraison à l’entrée arrière", "fragile — handle with care", "envío parcial, el resto a continuación", "Kunde holt selbst ab"]

    def vary(p):
        r = rng.random()
        if r < 0.3:
            return p.upper()
        if r < 0.6:
            return p.replace(" ", ", ", 1) + "."
        words = p.split()
        words[rng.randrange(len(words))] = rng.choice(["north", "30", "depot", "ltd"])
        return " ".join(words)

    out = []
    for _ in range(records):
        truth = {"vendor": rng.choice(vendors), "address": rng.choice(streets), "terms": rng.choice(terms), "note": rng.choice(notes),
                 "currency": rng.choice(["EUR", "USD", "GBP"]), "status": rng.choice(["paid", "open", "overdue"]), "kind": rng.choice(["invoice", "credit note"]),
                 "taxable": rng.random() < 0.5, "signed": rng.random() < 0.5,
                 "total": round(rng.uniform(10, 9000), 2), "tax": round(rng.uniform(1, 900), 2), "items": rng.randrange(1, 40)}
        cands = []
        for _c in range(n):
            d = {}
            for k, v in truth.items():
                r = rng.random()
                if r < 0.05:
                    v = None
                elif r < 0.25:
                    if isinstance(v, bool):
                        v = not v
                    elif isinstance(v, str):
                        v = vary(v) if " " in v and len(v) > 12 else v.upper()
                    elif isinstance(v, float):
                        v = round(v * rng.choice([1.0, 1.01, 10.0]), 2)
                    else:
                        v = v + rng.choice([0, 1])
                d[k] = v
            if nested:  # the same fields as an extraction schema would nest them (depth 3)
                d = {"vendor": {"name": d["vendor"], "location": {"address": d["address"], "currency": d["currency"]}},
                     "payment": {"terms": d["terms"], "status": d["status"], "signed": d["signed"]},
                     "amounts": {"total": d["total"], "tax": d["tax"], "taxable": d["taxable"]},
                     "kind": d["kind"], "note": d["note"], "items": d["items"]}
            if optional:
                d = _optional(rng, d, top=True)
            cands.append(json.dumps(d, ensure_ascii=not accents))
        out.append(cands)
    return out


def invoice_lines_texts(records, n, seed):
    """invoice_texts' schema with `items` as a LIST of 1..12 line items (a phrase description, a SKU enum, an int quantity, a
    float price): each candidate copies the record's line items with per-field noise, reorders them (probability 0.3), drops
    one (0.2) and adds one (0.1): the device path's list round."""
    import random
    rng = random.Random(seed + 1)
    descriptions = ["steel bolts m8 zinc plated", "hydraulic hose half inch", "industrial safety gloves large", "pallet wrap clear film",
                    "copper wire two millimetre", "led floodlight fifty watt", "cordless drill battery pack", "cable ties black 300mm"]
    skus = ["SKU-1001", "SKU-1002", "SKU-2040", "SKU-3300", "SKU-4712", "SKU-5000"]
    out = []
    for cands in invoice_texts(records, n, seed):
        truth = [{"description": rng.choice(descriptions), "sku": rng.choice(skus), "quantity": rng.randrange(1, 50),
                  "price": round(rng.uniform(0.5, 400), 2)} for _ in range(rng.randrange(1, 13))]
        lines_out = []
        for text in cands:
            d = json.loads(text)
            items = []
            for t in truth:
                it = dict(t)
                r = rng.random()
                if r < 0.1:
                    it["description"] = it["description"].upper()
                elif r < 0.15:
                    it["quantity"] = it["quantity"] + 1
                elif r < 0.2:
                    it["price"] = round(it["price"] * 1.01, 2)
                elif r < 0.23:
                    it["sku"] = None
                items.append(it)
            if len(items) > 1 and rng.random() < 0.2:
                del items[rng.randrange(len(items))]
            if rng.random() < 0.1:
                items.append({"description": rng.choice(descriptions), "sku": rng.choice(skus), "quantity": 1, "price": 9.99})
            if rng.random() < 0.3:
                rng.shuffle(items)
            d["items"] = items
            lines_out.append(json.dumps(d))
        out.append(lines_out)
    return out


def _optional(rng, d, top=False):
    items = [(k, _optional(rng, v) if isinstance(v, dict) else v) for k, v in d.items()]
    items = [(k, None if isinstance(v, dict) and rng.random() < P_NULL_SUB else v) for k, v in items
             if not (isinstance(v, dict) and rng.random() < P_MISSING_SUB)]
    if len(items) > 1 and rng.random() < P_DROP:
        del items[rng.randrange(len(items))]
    if top and rng.random() < P_EXTRA:
        items.append(("po_number", rng.choice(["PO-1001", "PO-1002", None])))
    if rng.random() < P_REORDER:
        rng.shuffle(items)
    return dict(items)


def workload_texts(workload, records, n, seed):
    """The candidate texts of an invoice workload."""
    if workload == "invoice_lines":
        return invoice_lines_texts(records, n, seed)
    return invoice_texts(records, n, seed, nested="nested" in workload, optional="optional" in workload, accents=workload == "unicode_invoice")


def batch_api(args):
    """consolidate_contents_batch on the workload's records: what the batch API (and, weighted, its Python planner for what the
    device path declines) does per call.  One JSON line, best of --reps after one warm-up call."""
    import random
    from k_llms_b200.utils import consolidation as C
    records = workload_texts(args.workload, args.records, args.n, 11)
    rng = random.Random(3)
    lps = [[[-rng.random() * 4, -rng.random()] for _ in r] for r in records] if args.weighted else None
    embed = lambda t: [[0.0] for _ in t]  # noqa: E731  (never called: no pair of long strings in these workloads)
    walls, counts = [], {}
    for i in range(args.reps + 1):
        counts = {}
        t0 = time.perf_counter()
        out = C.consolidate_contents_batch(records, get_openai_embeddings_from_text=embed, token_logprobs=lps, counts=counts)
        if i:
            walls.append(time.perf_counter() - t0)
    print(json.dumps({"what": "batch_api", "workload": args.workload, "weighted": args.weighted, "records": args.records, "n": args.n,
                      "best_s": round(min(walls), 4), "records_per_s": round(args.records / min(walls)), "counts": counts,
                      "example": str(out[0])[:80]}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", choices=["s32", "invoice", "invoice_nested", "invoice_optional", "invoice_nested_optional", "invoice_lines",
                                           "unicode_invoice"],
                    default="s32",
                    help="s32: the bench schema (enum / bool / number fields); invoice: 12 fields, 4 of them free text (medoid, K4); "
                         "invoice_nested: the same fields in nested objects (depth 3); *_optional: candidates that reorder, drop and add "
                         "keys and (nested) hold None or nothing for sub-objects; invoice_lines: `items` is a list of line items (list round); "
                         "unicode_invoice: invoice with accented, curly-quoted free text (KC_JSON_UNICODE)")
    ap.add_argument("--records", type=int, default=262144)
    ap.add_argument("--n", type=int, default=16)
    ap.add_argument("--reps", type=int, default=4)
    ap.add_argument("--chunk-mb", default="64")
    ap.add_argument("--streams", default="3")
    ap.add_argument("--pageable", action="store_true", help="input blob in ordinary (not page-locked) memory")
    ap.add_argument("--weighted", action="store_true", help="the likelihood-weighted variant (random candidate sums)")
    ap.add_argument("--no-lists", action="store_true", help="without JSON_LISTS: list records go to the host path (H1)")
    ap.add_argument("--no-unicode", action="store_true",
                    help="without JSON_UNICODE (here and in the batch API): non-ASCII records take the routes they took before it")
    ap.add_argument("--batch-api", action="store_true",
                    help="time consolidate_contents_batch (with --weighted: token logprobs, two per candidate) instead of the C-ABI call")
    args = ap.parse_args()
    if args.no_unicode:
        K.JSON_UNICODE = 0  # consolidation._native_consolidate reads it per call
    if args.batch_api:
        return batch_api(args)
    t0 = time.perf_counter()
    if args.workload != "s32":
        blob, off, _n = K.pack_texts(workload_texts(args.workload, args.records, args.n, 11), pinned=not args.pageable)
    else:
        blob, off = K.s32_texts_packed(args.records, args.n, 11, pinned=not args.pageable)
    gen_s = time.perf_counter() - t0
    flags = K.JSON_KEY_UNION | (0 if args.no_lists else K.JSON_LISTS) | K.JSON_UNICODE  # as the client functions call it
    seq = None
    if args.weighted:
        import numpy as np
        seq = (-np.random.default_rng(3).exponential(4.0, args.records * args.n)).astype(np.float32)
    for chunk in args.chunk_mb.split(","):
        for streams in args.streams.split(","):
            os.environ["KC_JSON_CHUNK_MB"], os.environ["KC_JSON_STREAMS"] = chunk, streams
            walls, stats = [], None
            for i in range(args.reps + 1):
                t0 = time.perf_counter()
                if seq is None:
                    res = K.consolidate_json_packed(blob, off, args.n, flags=flags)
                else:
                    res = K.consolidate_json_packed_weighted(blob, off, args.n, seq, flags=flags)
                dt = time.perf_counter() - t0
                stats = res.stats.as_dict()
                first = res.content(0)
                res.close()
                if i:
                    walls.append(dt)
            best = min(walls)
            print(json.dumps({"workload": args.workload, "weighted": args.weighted, "flags": flags, "records": args.records, "n": args.n,
                              "chunk_mb": int(chunk), "streams": int(streams),
                              "pinned_input": not args.pageable, "json_GB": round(stats["input_bytes"] / 1e9, 3),
                              "best_s": round(best, 4), "mean_s": round(sum(walls) / len(walls), 4),
                              "records_per_s": round(args.records / best), "n_device": stats["n_device"], "n_host": stats["n_host"],
                              "n_python": stats["n_python"], "json_GBps": round(stats["input_bytes"] / best / 1e9, 2),
                              "stats": {k: (round(v, 2) if isinstance(v, float) else v) for k, v in stats.items()},
                              "generate_s": round(gen_s, 1), "example": (first or "")[:80]}), flush=True)


if __name__ == "__main__":
    main()
