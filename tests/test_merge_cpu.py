"""`checkm merge`, CPU side: the library's merger.tsv row writer (host code, no device) against Python's own '%.2f', and
the oracle port against the merger.tsv files the reference's Merger wrote (tests/golden/merge/, made by
tests/golden/make_merge_goldens.py)."""
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN

MG = os.path.join(GOLDEN, 'merge')
HEADER_LINES = 1


@pytest.fixture(scope='module')
def golden():
    with open(os.path.join(MG, 'merge_goldens.json')) as f:
        return json.load(f)


def _rows(ids, p, s, n, pairs):
    from checkm_b200.engine import MERGE_PAIR_DTYPE
    from checkm_b200.merger import format_rows
    rec = np.zeros(len(pairs), dtype=MERGE_PAIR_DTYPE)
    for f, v in zip(('i', 'j', 'p', 's'), np.asarray(pairs, dtype=np.int64).reshape(-1, 4).T):
        rec[f] = v
    return format_rows(ids, p, s, n, rec).decode().splitlines(keepends=True)


def _python_row(ids, p, s, n, i, j, pm, sm):
    ci, ki = 100 * float(p[i]) / n[i], 100 * float(s[i] - p[i]) / n[i]
    cj, kj = 100 * float(p[j]) / n[j], 100 * float(s[j] - p[j]) / n[j]
    c, k = 100 * float(pm) / n[j], 100 * float(sm - pm) / n[j]
    dc, dk = c - max(ci, cj), k - max(ki, kj)
    return '%s\t%s\t%.2f\t%.2f\t%.2f\t%.2f\t%.2f\t%.2f\t%.2f\t%.2f\t%.2f\n' % (ids[i], ids[j], ci, ki, cj, kj, dc, dk, dc - dk, c, k)


def test_writer_prints_as_python_for_every_ratio():
    """Every (p, N) with 0 <= p <= N <= 2000 as the completeness of bin i (s = p) and as the merged completeness of a pair
    (bin j has N markers, p_j = 0), so the deltas between them are printed too."""
    N = np.concatenate([np.full(k + 1, k, dtype=np.int64) for k in range(1, 2001)])
    P = np.concatenate([np.arange(k + 1, dtype=np.int64) for k in range(1, 2001)])
    m = len(N)
    ids = ['a%d' % x for x in range(m)] + ['b%d' % x for x in range(m)]
    p = np.concatenate([P, np.zeros(m, np.int64)])
    s = np.concatenate([P + (P % 7), np.zeros(m, np.int64)])
    n = np.concatenate([np.maximum(N, 1), np.maximum(N[::-1], 1)])
    q = np.arange(m)
    pm = np.minimum(P[::-1], n[m + q])                       # merged completeness p / N_j
    pairs = np.stack([q, m + q, pm, pm + (q % 5)], axis=1)
    got = _rows(ids, p, s, n, pairs)
    want = [_python_row(ids, p, s, n, i, j, a, b) for i, j, a, b in pairs.tolist()]
    assert got == want


def test_writer_prints_as_python_for_random_tuples():
    rng = np.random.default_rng(7)
    nb, m = 4000, 1_000_000
    ids = ['bin_%d' % x for x in range(nb)]
    n = rng.integers(1, 6000, size=nb)
    p = (rng.random(nb) * (n + 1)).astype(np.int64).clip(0, n)
    s = p + rng.integers(0, 1 << 16, size=nb) * (p > 0)
    i = rng.integers(0, nb, size=m)
    j = rng.integers(0, nb, size=m)
    pm = np.minimum(p[i] + p[j], n[j] + rng.integers(0, 3, size=m))
    sm = s[i] + s[j]
    pairs = np.stack([i, j, pm, sm], axis=1)
    got = _rows(ids, p, s, n, pairs)
    want = [_python_row(ids, p, s, n, *t) for t in pairs.tolist()]
    assert got == want


def _cases(golden):
    for case, g in golden['cases'].items():
        for which, e in g.items():
            cn = {b: {m: c for m, c in zip(e['markers'], row) if c} for b, row in zip(e['bins'], e['copy_numbers'])}
            nm = dict(zip(e['bins'], e['n_markers']))
            for label, thr in e['thresholds'].items():
                yield (case, which, label), e, cn, nm, thr


def test_oracle_matches_every_golden(golden):
    from oracle.merge_oracle import merge_pairs
    n = 0
    for key, e, cn, nm, thr in _cases(golden):
        lines, _ = merge_pairs(e['bins'], cn, nm, e['markers'], *thr)
        assert e['tsv'][key[2]].splitlines(keepends=True)[HEADER_LINES:] == lines, key
        n += 1
    assert n == 16


def test_writer_matches_every_golden(golden):
    """The pairs the oracle keeps, written by the library's writer from (p, s, N) alone."""
    from oracle.merge_oracle import merge_pairs
    for key, e, cn, nm, thr in _cases(golden):
        counts = np.array(e['copy_numbers'], dtype=np.int64)
        p, s = (counts > 0).sum(1), counts.sum(1)
        _, pairs = merge_pairs(e['bins'], cn, nm, e['markers'], *thr)
        rec = [(i, j, int(((counts[i] > 0) | (counts[j] > 0)).sum()), s[i] + s[j]) for i, j in pairs]
        got = _rows(e['bins'], p, s, np.array(e['n_markers']), rec)
        assert e['tsv'][key[2]].splitlines(keepends=True)[HEADER_LINES:] == got, key
