"""Seeded synthetic FCMA workloads (host side, numpy only).

The recipe is the one fixed in SURVEY.md §8(d): per epoch ``RandomState(1234567890 + e)``
Gaussian ``[T, V]`` data, a planted common time course added to the first ``V // 100`` voxels of
odd-labelled epochs, then the reference normalisation exactly as
``brainiak.fcma.preprocessing._separate_epochs`` (reference preprocessing.py:80-84):
``zscore(axis=0, ddof=0)`` -> ``nan_to_num`` -> ``/ sqrt(T)``, C-contiguous float32.
"""
import math

import numpy as np

SEED = 1234567890


def make_labels(E):
    """labels = [e % 2]: every subject block of ``eps`` (even) epochs is balanced."""
    return [e % 2 for e in range(E)]


def raw_epoch(e, T, V, seed=SEED, signal=0.6, informative=None):
    """Un-normalised epoch ``[T, V]`` float32 (the input of the normalise prologue)."""
    rng = np.random.RandomState(seed + e)
    m = rng.randn(T, V).astype(np.float32)
    if informative is None:
        informative = V // 100
    if e % 2 == 1 and informative > 0:
        common = rng.randn(T, 1).astype(np.float32)
        m[:, :informative] += np.float32(signal) * common
    return m


def normalize_epoch(m):
    """Reference preprocessing.py:80-84 on one ``[T, V]`` block (float32 numpy arithmetic)."""
    m = np.asarray(m, dtype=np.float32)
    mn = m.mean(axis=0, keepdims=True)
    sd = m.std(axis=0, ddof=0, keepdims=True)
    with np.errstate(invalid="ignore", divide="ignore"):
        z = (m - mn) / sd
    z = np.nan_to_num(z)
    return np.ascontiguousarray(z / np.float32(math.sqrt(m.shape[0])), dtype=np.float32)


def make_epochs(V, T, E, seed=SEED, normalized=True, signal=0.6, informative=None):
    """Returns ``(raw_data, labels)``: ``raw_data`` is a list of E float32 ``[T, V]`` arrays."""
    data = []
    for e in range(E):
        m = raw_epoch(e, T, V, seed=seed, signal=signal, informative=informative)
        data.append(normalize_epoch(m) if normalized else m)
    return data, make_labels(E)


def make_two_masks(V, V2, T, E, seed=SEED):
    """Two-mask workload: ``raw_data`` ``[T, V]`` and ``raw_data2`` ``[T, V2]`` per epoch."""
    d1, labels = make_epochs(V, T, E, seed=seed)
    d2, _ = make_epochs(V2, T, E, seed=seed + 7919)
    return d1, d2, labels


def make_dyadic_epochs(V, T, E, seed=SEED, informative=None):
    """Like ``make_epochs`` (planted common time course in the first ``informative`` voxels of odd-labelled epochs), but
    every value is a multiple of 1/32 with magnitude at most 5/32 and ``T <= 40``: every product and every partial sum of
    a correlation is exact in fp32, so any summation order gives the same r, bit for bit (|r| < 1).  Not normalised."""
    if T > 40:
        raise ValueError("T must be at most 40 for exact correlations")
    if informative is None:
        informative = max(1, V // 6)
    data = []
    for e in range(E):
        rng = np.random.RandomState(seed + e)
        m = rng.randint(-3, 4, size=(T, V))
        if e % 2 == 1:
            m[:, :informative] += rng.randint(-2, 3, size=(T, 1))
        data.append(np.ascontiguousarray(m.astype(np.float32) / np.float32(32)))
    return data, make_labels(E)
