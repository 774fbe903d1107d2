"""Evaluate word vectors: nearest words, analogies, word-similarity correlation (word2vec's ``distance``,
``word-analogy`` / ``compute-accuracy``, and the WS-353 protocol).

    python -m multiverso_b200.apps.wordembedding_eval -vectors vec.bin -binary 1 \
        -analogy questions-words.txt -threshold 30000 -similarity ws353.txt -neighbours king,paris -k 10

* ``-vectors <file> -binary <0|1>``: the word2vec text or binary file written by ``WordEmbedding.save_embedding``
  and by the native ``wordembedding`` binaries.
* ``-analogy <file>``: ``: section`` headers and ``a b c d`` lines. A question counts as correct when the row
  nearest to unit(b) - unit(a) + unit(c), a, b and c excluded, is d. Only the first ``-threshold`` words
  (default 30000, as compute-accuracy) are candidates; a question with a word out of the vocabulary or beyond
  the threshold is skipped. Words match case-sensitively (compute-accuracy upper-cases everything).
* ``-similarity <file>``: ``w1 w2 score`` lines, ``#`` comments; Spearman rank correlation (average ranks for
  ties) between the scores and the vectors' cosines.
* ``-neighbours w1,w2,...`` with ``-k``: the nearest words of each, the word itself excluded.
* ``-device cuda|cpu``: where the search runs (default: the GPU when there is one, else the host
  implementation of the same search).

The result is one JSON line.
"""
from __future__ import annotations

import json
import sys
from typing import Dict, List, Optional, Tuple

import numpy as np

FLAG_HELP = """-vectors <file> -binary <0|1> -analogy <file> -threshold <int> -similarity <file>
-neighbours <w1,w2,...> -k <int> -device <cuda|cpu>"""


def load_vectors(path: str, binary: bool) -> Tuple[List[str], np.ndarray]:
    """word2vec text / binary vector file: header ``V D``, then per word its name and D floats (binary: a
    space, 4 D bytes of little-endian fp32, an optional newline)."""
    with open(path, "rb") as f:
        V, D = map(int, f.readline().split())
        words: List[str] = []
        vecs = np.empty((V, D), dtype=np.float32)
        if binary:
            data = f.read()
            p = 0
            for i in range(V):
                while p < len(data) and data[p:p + 1] in (b"\n", b" "):
                    p += 1
                sp = data.index(b" ", p)
                words.append(data[p:sp].decode(errors="replace"))
                p = sp + 1
                if p + 4 * D > len(data):
                    raise ValueError(f"{path}: truncated at word {i} of {V}")
                vecs[i] = np.frombuffer(data, dtype="<f4", count=D, offset=p)
                p += 4 * D
        else:
            for i in range(V):
                parts = f.readline().split()
                if len(parts) != D + 1:
                    raise ValueError(f"{path}: line {i + 2} has {len(parts) - 1} values, expected {D}")
                words.append(parts[0].decode(errors="replace"))
                vecs[i] = np.array(parts[1:], dtype=np.float32)
    return words, vecs


def read_questions(path: str) -> List[Tuple[str, List[str]]]:
    """``questions-words.txt`` format: (section, [a, b, c, d]) per question line."""
    out, section = [], ""
    with open(path, encoding="utf-8", errors="replace") as f:
        for line in f:
            s = line.strip()
            if not s:
                continue
            if s.startswith(":"):
                section = s[1:].strip()
                continue
            parts = s.split()
            if len(parts) == 4:
                out.append((section, parts))
    return out


def read_pairs(path: str) -> List[Tuple[str, str, float]]:
    """``w1 w2 score`` lines; ``#`` starts a comment."""
    out = []
    with open(path, encoding="utf-8", errors="replace") as f:
        for line in f:
            s = line.split("#", 1)[0].split()
            if len(s) >= 3:
                out.append((s[0], s[1], float(s[2])))
    return out


def _average_ranks(x: np.ndarray) -> np.ndarray:
    order = np.argsort(x, kind="mergesort")
    _, start, counts = np.unique(x[order], return_index=True, return_counts=True)
    ranks = np.empty(len(x), dtype=np.float64)
    ranks[order] = np.repeat(start + (counts + 1) / 2.0, counts)
    return ranks


def spearman(x, y) -> float:
    """Spearman rank correlation with average ranks for ties (NaN for fewer than 2 pairs or a constant side)."""
    x, y = np.asarray(x, dtype=np.float64), np.asarray(y, dtype=np.float64)
    if len(x) < 2:
        return float("nan")
    rx, ry = _average_ranks(x), _average_ranks(y)
    rx -= rx.mean()
    ry -= ry.mean()
    den = np.sqrt((rx * rx).sum() * (ry * ry).sum())
    return float((rx * ry).sum() / den) if den > 0 else float("nan")


class Evaluator:
    """The vectors as a search table: on the GPU the fused top-k kernel over a CUDA tensor, on the host the
    reference implementation over a CPU tensor."""

    def __init__(self, words: List[str], vecs: np.ndarray, device: str):
        import torch
        self.words, self.device = words, device
        self.index: Dict[str, int] = {}
        for i, w in enumerate(words):
            self.index.setdefault(w, i)
        D = vecs.shape[1]
        pitch = (D + 3) // 4 * 4                  # 16-byte rows for TMA; the padding columns are not compared
        t = torch.zeros(len(words), pitch, dtype=torch.float32)
        t[:, :D] = torch.from_numpy(vecs)
        self.table = t.to(device)
        self.D = D

    def rows(self, ids):
        import torch
        return self.table[torch.as_tensor(ids, dtype=torch.int64, device=self.table.device), :self.D]

    def analogy(self, a, b, c, threshold: int):
        """Top-1 answers (ids) of 3CosAdd questions over rows [0, threshold)."""
        import torch
        from ..ops.topk import analogy_queries, take_excluding, topk_cosine
        if len(a) == 0:
            return np.zeros(0, dtype=np.int64)
        q = analogy_queries(self.rows(a), self.rows(b), self.rows(c))
        s, i = topk_cosine(self.table, q, 4, rows=min(threshold, len(self.words)))
        ex = torch.as_tensor(np.stack([a, b, c], 1), device=i.device)
        return take_excluding(s, i, ex, 1)[1][:, 0].cpu().numpy()

    def neighbours(self, ids, k: int):
        import torch
        from ..ops.topk import check_k, take_excluding, topk_cosine
        k = check_k(k, 1, "-neighbours -k")
        s, i = topk_cosine(self.table, self.rows(ids), k + 1)
        ex = torch.as_tensor(np.asarray(ids)[:, None], device=i.device)
        s, i = take_excluding(s, i, ex, k)
        return s.cpu().numpy(), i.cpu().numpy()


def eval_analogy(ev: Evaluator, questions, threshold: int) -> dict:
    sections: Dict[str, dict] = {}
    ids, secs, skipped = [], [], 0
    for sec, ws in questions:
        sections.setdefault(sec, {"correct": 0, "seen": 0})
        ix = [ev.index.get(w, -1) for w in ws]
        if min(ix) < 0 or max(ix) >= threshold:
            skipped += 1
            continue
        ids.append(ix)
        secs.append(sec)
    arr = np.asarray(ids, dtype=np.int64).reshape(-1, 4)
    ans = ev.analogy(arr[:, 0], arr[:, 1], arr[:, 2], threshold)
    ok = ans == arr[:, 3]
    for sec, good in zip(secs, ok):
        sections[sec]["seen"] += 1
        sections[sec]["correct"] += int(good)
    for d in sections.values():
        d["accuracy"] = d["correct"] / d["seen"] if d["seen"] else None
    seen = len(secs)
    return {"sections": sections, "correct": int(ok.sum()), "seen": seen, "skipped": skipped,
            "questions": len(questions), "threshold": threshold,
            "accuracy": float(ok.sum()) / seen if seen else None}


def eval_similarity(ev: Evaluator, pairs) -> dict:
    human, model, skipped = [], [], 0
    for w1, w2, score in pairs:
        i1, i2 = ev.index.get(w1, -1), ev.index.get(w2, -1)
        if i1 < 0 or i2 < 0:
            skipped += 1
            continue
        v1 = ev.rows([i1]).double().cpu().numpy()[0]
        v2 = ev.rows([i2]).double().cpu().numpy()[0]
        n = np.linalg.norm(v1) * np.linalg.norm(v2)
        human.append(score)
        model.append(float(v1 @ v2 / n) if n > 0 else 0.0)
    rho = spearman(human, model)
    return {"spearman": None if np.isnan(rho) else rho, "pairs": len(human), "skipped": skipped}


def parse_args(argv: List[str]) -> dict:
    """``-flag value`` pairs like the applications' Option::ParseArgs."""
    o = {"vectors": None, "binary": 0, "analogy": None, "threshold": 30000, "similarity": None,
         "neighbours": None, "k": 10, "device": None}
    conv = {"binary": int, "threshold": int, "k": int}
    i = 0
    while i < len(argv):
        a = argv[i]
        if a.startswith("-") and a[1:] in o and i + 1 < len(argv):
            o[a[1:]] = conv.get(a[1:], str)(argv[i + 1])
            i += 2
        else:
            raise SystemExit(f"unknown or incomplete flag {a!r}; usage: wordembedding_eval {FLAG_HELP}")
    return o


def run(argv: List[str]) -> dict:
    import torch
    o = parse_args(argv)
    if not o["vectors"]:
        print("usage: wordembedding_eval " + FLAG_HELP)
        return {}
    device = o["device"] or ("cuda" if torch.cuda.is_available() else "cpu")
    words, vecs = load_vectors(o["vectors"], bool(o["binary"]))
    ev = Evaluator(words, vecs, device)
    res: dict = {"vectors": len(words), "dim": ev.D, "device": device}
    if o["analogy"]:
        res["analogy"] = eval_analogy(ev, read_questions(o["analogy"]), o["threshold"])
    if o["similarity"]:
        res["similarity"] = eval_similarity(ev, read_pairs(o["similarity"]))
    if o["neighbours"]:
        qs = [w for w in o["neighbours"].split(",") if w]
        known = [w for w in qs if w in ev.index]
        res["neighbours"] = {w: None for w in qs}
        if known:
            s, i = ev.neighbours([ev.index[w] for w in known], o["k"])
            for r, w in enumerate(known):
                res["neighbours"][w] = [[words[j], round(float(v), 6)] for v, j in zip(s[r], i[r]) if j >= 0]
    print(json.dumps(res), flush=True)
    return res


if __name__ == "__main__":
    run(sys.argv[1:])
