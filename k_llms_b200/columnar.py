"""Host prologue / epilogue of the CUDA consensus path: flatten candidate objects into columnar groups,
run K1/K2 once over ALL groups of ALL records, rebuild the (value, confidence) trees.

The recursion mirrors the reference dispatcher `consensus_values` (consensus_utils.py:1376-1454, "cu") but
instead of computing a scalar field it RECORDS it as a group:

  * vote group    (cu:1405-1411 -> voting_consensus cu:936-982): cells = local dictionary codes of the
    processed values (`sanitize_value(v)` cu:925-933 for strings, `v or False` cu:956 for bools), None = -1
  * numeric group (cu:1443-1453 -> consensus_as_primitive cu:1098-1219): cells = float(v); None, bools,
    strings, nan/inf are tagged so the kernel counts them exactly as the reference does (cu:1100-1114)

The shape of the result (dict keys in first-seen order cu:1281-1282, list lengths cu:1332-1341, the
parent_valid_frac products cu:1418,1433,1444) depends only on the input structure, so it is fixed while
planning; the GPU fills in the leaves.  Multi-word string fields (the similarity medoid, cu:1221-1237) are recorded as
medoid groups for K4 when every pair is a Levenshtein pair inside the kernel's contract (`Plan._medoid_on_device`);
mixed payloads and the other similarity methods are computed by `k_llms_b200.utils.similarity` on the host.
"""
from __future__ import annotations

import math
import re
from typing import Any, Callable, List, Optional, Sequence, Tuple

import numpy as np

from . import _native

MAX_CANDIDATES = _native.MAX_CANDIDATES
SKIPPED_KEY_MARKERS = ("reasoning___", "source___")  # cu:1287

_F64_NONE = np.array([_native.F64_NONE_BITS], dtype=np.uint64).view(np.float64)[0]
_F64_ABSENT = np.array([_native.F64_ABSENT_BITS], dtype=np.uint64).view(np.float64)[0]


# ----------------------------------------------------------------------------- sanitising (cu:925-933)

try:  # a dependency of the package (pyproject.toml), as of the reference (requirements.txt); ASCII input never reaches it
    from unidecode import unidecode as _unidecode  # type: ignore
except Exception:  # pragma: no cover - depends on the image
    _unidecode = None


def _fold_non_ascii(s: str) -> str:
    """unidecode(s) (cu:931).  Without the Unidecode package the vote classes of non-ASCII text would differ from the
    reference's ('Straße' / 'Strasse' share a class under unidecode), so this fails loudly instead of guessing — unless
    KLLMS_B200_ALLOW_NFKD=1 opts into NFKD folding (a documented deviation: combining marks are dropped, ß ø æ CJK are not
    transliterated)."""
    if _unidecode is not None:
        return _unidecode(s)
    import os
    if os.environ.get("KLLMS_B200_ALLOW_NFKD") != "1":
        raise ImportError("non-ASCII text needs the Unidecode package (a dependency of k_llms_b200, see pyproject.toml) to be "
                          "sanitised like the reference does; install it, or set KLLMS_B200_ALLOW_NFKD=1 to accept NFKD folding")
    import unicodedata
    return "".join(ch for ch in unicodedata.normalize("NFKD", s) if not unicodedata.combining(ch))


def _normalize(text: str) -> str:
    """normalize_string (cu:660-673): keep ASCII alphanumerics, lower-case."""
    return "".join(ch for ch in text if ch.isascii() and ch.isalnum()).lower() if text else ""


_NOT_ALNUM = re.compile(r"[^a-zA-Z0-9]")


def sanitize_value(v: Any) -> str:
    """str() -> lower -> drop spaces -> unidecode -> keep [a-zA-Z0-9]  (cu:925-933)."""
    s = str(v).lower().replace(" ", "")
    if not s.isascii():
        s = _fold_non_ascii(s)
    return _NOT_ALNUM.sub("", s)


# ----------------------------------------------------------------------------- plan nodes


class _Const:
    __slots__ = ("value", "conf")

    def __init__(self, value, conf):
        self.value, self.conf = value, conf


class _VoteLeaf:
    __slots__ = ("row", "cells", "pvf", "where")

    def __init__(self, row: int, cells: list, pvf: float, where: Optional[dict] = None):
        self.row, self.cells, self.pvf = row, cells, pvf  # cells[i] = value returned when cell i wins
        self.where = where  # weighted plans: candidate position of a cell -> its index in `cells`


class _NumLeaf:
    __slots__ = ("row", "cells", "pvf")

    def __init__(self, row: int, cells: list, pvf: float):
        self.row, self.cells, self.pvf = row, cells, pvf


class _MedoidLeaf:
    __slots__ = ("row", "cells", "pvf")

    def __init__(self, row: int, cells: list, pvf: float):
        self.row, self.cells, self.pvf = row, cells, pvf


class _DictNode:
    __slots__ = ("children",)

    def __init__(self, children: dict):
        self.children = children


class _ListNode:
    __slots__ = ("children",)

    def __init__(self, children: list):
        self.children = children


class Plan:
    """Leaf groups of one or many records, ready for one K1, one K2 and one K4 launch.

    Weighted plans (`weighted=True`, DESIGN.md §5, likelihood-weighted consensus): every record starts with `begin_record(sums)`,
    the fp32 sequence logprobs of its candidates.  Vote cells then stay at their CANDIDATE's position (a candidate that is not a
    dict / list at some node is an absent cell below it, instead of being compacted away), each vote row remembers its record,
    and `run()` votes with one launch of K3b over ragged records (kc_weighted_vote_groups_i8) instead of K1.  Everything else —
    numeric clusters, medoids, parent_valid_frac, key order — is planned exactly as in count mode."""

    def __init__(self, n: int, allow_none_as_candidate: bool, rel_eps: float, abs_eps: float, host_primitive: Callable,
                 numeric_branch: bool = True, weighted: bool = False):
        if n > MAX_CANDIDATES:
            raise ValueError(f"{n} candidates per request: k_llms_b200 consolidates at most {MAX_CANDIDATES} (one kernel row per "
                             "field holds every candidate; the package has no CPU path to fall back to)")
        # False: the reference's ASYNC dispatcher, whose primitive has no numeric clustering (cu:1638-1688): numbers take the
        # similarity medoid like any other non-enum value
        self.numeric_branch = numeric_branch
        self.n = max(n, 1)
        self.allow_none = allow_none_as_candidate
        self.rel_eps, self.abs_eps = rel_eps, abs_eps
        self.host_primitive = host_primitive
        self.vote_rows: List[List[int]] = []
        self.num_rows: List[List[float]] = []
        self.medoid_groups: List[List[str]] = []  # normalised strings of the groups K4 handles
        self.string_method = "embeddings"         # set by the caller (ConsensusSettings.string_similarity_method)
        self.weighted = weighted
        self.vote_record: List[int] = []          # weighted: the record of each vote row
        self.seq_logprobs: List[List[float]] = []  # weighted: the candidates' sums of each record, padded to n

    def begin_record(self, seq_logprobs: Sequence[float]) -> None:
        """Weighted plans: the records' candidate sums, in the order of the add() calls that plan them."""
        if len(seq_logprobs) > self.n:
            raise ValueError(f"{len(seq_logprobs)} sequence logprobs for at most {self.n} candidates")
        # a candidate the record does not have weighs nothing, and does not shift the record's maximum (kc_weighted_vote_groups_i8)
        self.seq_logprobs.append([float(s) for s in seq_logprobs] + [-3.0e38] * (self.n - len(seq_logprobs)))

    # -- leaves ---------------------------------------------------------------------------------------
    def _vote(self, values: Sequence[Any], pvf: float, pos: Optional[Sequence[int]] = None) -> _VoteLeaf:
        first = next(v for v in values if v is not None)
        codes: List[int] = []
        table: dict = {}
        if isinstance(first, bool):  # cu:954-958: None and every falsy value become False
            cells = [v or False for v in values]
            for k in cells:
                codes.append(table.setdefault(k, len(table)))
        else:
            cells = list(values)
            for v in values:
                if v is None and not self.allow_none:
                    codes.append(_native.CODE_NONE)  # cu:964: None does not vote
                else:
                    k = None if v is None else sanitize_value(v)
                    codes.append(table.setdefault(k, len(table)))
        where = None
        if pos is not None:  # weighted: cell i at candidate pos[i], the candidates filtered out above are absent
            row = [_native.CODE_ABSENT] * self.n
            for p, c in zip(pos, codes):
                row[p] = c
            codes, where = row, {p: i for i, p in enumerate(pos)}
            self.vote_record.append(len(self.seq_logprobs) - 1)
        codes.extend([_native.CODE_ABSENT] * (self.n - len(codes)))
        self.vote_rows.append(codes)
        return _VoteLeaf(len(self.vote_rows) - 1, cells, pvf, where)

    def _numeric(self, values: Sequence[Any], pvf: float) -> _NumLeaf:
        row: List[float] = []
        for v in values:
            if v is None:
                row.append(_F64_NONE)
            elif isinstance(v, bool) or not isinstance(v, (int, float)):
                row.append(math.nan)  # present, counted in `total`, never clustered (cu:1106-1108)
            else:
                try:
                    row.append(float(v))  # non-finite floats are dropped by the kernel (cu:1111)
                except OverflowError:
                    row.append(math.nan)  # cu:1113-1114
        row.extend([_F64_ABSENT] * (self.n - len(row)))
        self.num_rows.append(row)
        return _NumLeaf(len(self.num_rows) - 1, list(values), pvf)

    # -- dispatcher (cu:1376-1454) ----------------------------------------------------------------------
    def add(self, values: Sequence[Any], pvf: float, embed: Optional[Callable], pos: Optional[Sequence[int]] = None):
        """Plan one record's candidate values (or, recursively, one node's).  pos (weighted plans): the candidate position of
        each value; a weighted record's top-level call leaves it to default to 0..len(values)-1."""
        if self.weighted and pos is None:
            if len(self.seq_logprobs) == 0:
                raise ValueError("a weighted plan needs begin_record(seq_logprobs) before each record")
            pos = range(len(values))
        if not values:
            return _Const(None, pvf)  # cu:1395-1396
        live = [v for v in values if v is not None]
        if not live:
            return _Const(None, 0.0)  # cu:1401-1402
        head = live[0]
        if isinstance(head, (str, bool)) and all(len(str(v).strip().split()) < 3 for v in live):
            return self._vote(values, pvf, pos)  # cu:1405-1411
        if isinstance(head, dict):  # cu:1414-1426 -> consensus_dict cu:1269-1306
            keep = [i for i, v in enumerate(values) if isinstance(v, dict)]
            dicts = [values[i] for i in keep]
            sub_pos = None if pos is None else [pos[i] for i in keep]
            sub = pvf * (len(dicts) / len(values))
            keys: dict = {}
            for d in dicts:
                for k in d:
                    keys.setdefault(k, None)
            children = {}
            for k in keys:
                if any(mark in k for mark in SKIPPED_KEY_MARKERS):
                    continue
                children[k] = self.add([d.get(k) for d in dicts], sub, embed, sub_pos)
            return _DictNode(children)
        if isinstance(head, list):  # cu:1429-1441 -> consensus_list cu:1309-1352
            keep = [i for i, v in enumerate(values) if isinstance(v, list)]
            lists = [values[i] for i in keep]
            sub_pos = None if pos is None else [pos[i] for i in keep]
            sub = pvf * (len(lists) / len(values))
            longest = max(len(l) for l in lists)
            return _ListNode([self.add([l[i] if i < len(l) else None for l in lists], sub, embed, sub_pos) for i in range(longest)])
        if embed is None:  # cu:1445-1446
            raise ValueError("sync_get_openai_embeddings_from_text is required for primitive consensus")
        try:
            numeric_like = isinstance(type(head)(), (int, float))  # cu:1099
        except Exception:
            numeric_like = False
        if self.numeric_branch and (numeric_like or all(isinstance(v, (int, float)) for v in live)):
            # the kernel applies the None-stripping and len(values) bookkeeping of cu:1444 / cu:1082-1086 itself
            return self._numeric(values, pvf)
        sub = pvf * (len(live) / len(values))  # cu:1444
        if len(live) == 1:
            return _Const(live[0], sub * (1 / 1))  # cu:1085-1086
        if self._medoid_on_device(live):
            self.medoid_groups.append([_normalize(s) for s in live])
            return _MedoidLeaf(len(self.medoid_groups) - 1, live, sub)
        value, conf = self.host_primitive(live, sub, embed)  # similarity medoid on the host, cu:1221-1237
        return _Const(value, conf)

    def _medoid_on_device(self, live: Sequence[Any]) -> bool:
        """K4 takes groups of plain ASCII strings: methods 'jaccard' and 'hamming' always; 'levenshtein' when every pair has a
        <= 64-character side; 'embeddings' where, further, no two strings are both longer than 50 characters (cu:813 would ask
        the embeddings service for those)."""
        if self.string_method not in ("levenshtein", "embeddings", "jaccard", "hamming") or len(live) > MAX_CANDIDATES:
            return False
        if not all(isinstance(v, str) and v.isascii() for v in live):
            return False
        if self.string_method == "embeddings" and sum(1 for v in live if len(v) > 50) > 1:
            return False
        lens = [len(_normalize(v)) for v in live]
        if self.string_method in ("jaccard", "hamming"):  # character sets / position-wise mismatches: no pattern-length contract
            return max(lens) <= 2000
        return sum(1 for l in lens if l > 64) <= 1 and max(lens) <= 2000

    # -- device ----------------------------------------------------------------------------------------
    def run(self, device=None):
        """One K1, one K2 and one K4 launch over every recorded group; returns numpy result columns."""
        import torch
        if not torch.cuda.is_available():
            raise RuntimeError("k_llms_b200: no CUDA device — the consensus hot path has no CPU fallback")
        dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        out = {}
        if self.vote_rows and self.weighted:  # K3b over ragged records: every cell is a local code < 64, so int8 holds it
            codes = torch.from_numpy(np.asarray(self.vote_rows, dtype=np.int8)).to(dev)
            rec = torch.from_numpy(np.asarray(self.vote_record, dtype=np.int32)).to(dev)
            seq = torch.from_numpy(np.asarray(self.seq_logprobs, dtype=np.float32).reshape(-1, self.n)).to(dev)
            _, meta, weight = _native.weighted_vote_groups(codes, rec, seq)
            out["vote_meta"] = meta.cpu().numpy().view(np.uint32)
            out["vote_weight"] = weight.cpu().numpy()
        elif self.vote_rows:
            codes = torch.from_numpy(np.asarray(self.vote_rows, dtype=np.int32)).to(dev)
            _, meta = _native.vote(codes, None)
            out["vote_meta"] = meta.cpu().numpy().view(np.uint32)
        if self.num_rows:
            vals = torch.from_numpy(np.asarray(self.num_rows, dtype=np.float64)).to(dev)
            value, meta = _native.numeric(vals, self.rel_eps, self.abs_eps)
            out["num_value"] = value.cpu().numpy()
            out["num_meta"] = meta.cpu().numpy().view(np.uint32)
        if self.medoid_groups:
            blobs, str_off, grp_off = [], [0], [0]
            for grp in self.medoid_groups:
                for s in grp:
                    b = s.encode("ascii")
                    blobs.append(b)
                    str_off.append(str_off[-1] + len(b))
                grp_off.append(grp_off[-1] + len(grp))
            chars = np.frombuffer(b"".join(blobs) or b"\0", dtype=np.uint8).copy()
            idx, avg = _native.medoid_str(torch.from_numpy(chars).to(dev), torch.tensor(str_off, dtype=torch.int32, device=dev),
                                          torch.tensor(grp_off, dtype=torch.int32, device=dev),
                                          max_group=max(len(grp) for grp in self.medoid_groups), method=self.string_method)
            out["medoid_idx"], out["medoid_avg"] = idx.cpu().numpy(), avg.cpu().numpy()
        return out

    # -- epilogue --------------------------------------------------------------------------------------
    @staticmethod
    def _fields(m: int) -> Tuple[int, int, int, int, int]:
        return m & 0x3F, (m >> 6) & 0x7F, (m >> 13) & 0x7F, (m >> 20) & 0x7F, (m >> 27) & 0x1F

    def materialise(self, node, res) -> Tuple[Any, Any]:
        if isinstance(node, _Const):
            return node.value, node.conf
        if isinstance(node, _DictNode):
            val, conf = {}, {}
            for k, child in node.children.items():
                val[k], conf[k] = self.materialise(child, res)
            return val, conf
        if isinstance(node, _ListNode):
            pairs = [self.materialise(c, res) for c in node.children]
            return [p[0] for p in pairs], [p[1] for p in pairs]
        if isinstance(node, _MedoidLeaf):  # cu:1233-1237
            return node.cells[int(res["medoid_idx"][node.row])], round(node.pvf * float(res["medoid_avg"][node.row]), 5)
        if isinstance(node, _VoteLeaf):
            idx, support, _nn, present, flags = self._fields(int(res["vote_meta"][node.row]))
            if not flags & _native.FLAG_HAS_VALUE:  # cannot happen for a planned vote group (>= 1 voter)
                return None, (node.pvf if present == 0 else 0.0)
            if node.where is not None:  # weighted (DESIGN.md §5): idx is a candidate position; pvf x the winner's share of the weight
                return node.cells[node.where[idx]], round(node.pvf * float(res["vote_weight"][node.row]), 5)
            return node.cells[idx], round(node.pvf * (support / present), 5)  # cu:971,973,982
        idx, support, nn, present, flags = self._fields(int(res["num_meta"][node.row]))
        if flags & _native.FLAG_HAS_VALUE:
            if flags & _native.FLAG_SINGLE:
                return node.cells[idx], node.pvf * (1 / present) * (1 / 1)  # cu:1444, cu:1085-1086
            return float(res["num_value"][node.row]), round(support / nn, 5)  # cu:1176-1178,1217-1219
        if flags & _native.FLAG_NO_FINITE:
            return None, node.pvf * (nn / present)  # cu:1444, cu:1115-1116
        return None, (node.pvf if present == 0 else 0.0)
