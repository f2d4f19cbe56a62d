"""Rotation-only RANSAC of an image pair in numpy: the CPU restatement that opensfm_b200/csrc/rotransac.cu is checked
against.

What it restates (pyrobust's `ransac_relative_rotation` with RANSAC scoring, as `compute_image_pairs` calls it through
`multiview.relative_pose_ransac_rotation_only`, then `_two_view_rotation_inliers` and `pairwise_reconstructability`):

  * the sample stream: a std::mt19937 seeded with 42, restarted for every pair; an index in [0, n) is drawn from its
    32-bit outputs by libstdc++'s `uniform_int_distribution<unsigned long>` (GCC 13: Lemire's product with
    rejection); a draw that repeats an index already in the sample is drawn again;
  * 3-point samples, up to `iterations` of them; a model's error on row i is 1 - (M b1_i) . b2_i, an inlier when its
    absolute value is below 1 - cos(threshold); a model replaces the best one when it has at least as many inliers;
  * local optimisation whenever a model ties or beats the best with at least 3 inliers: 10 rounds, each drawing
    max(min(12, floor(inliers / 2)), 3) positions of the best model's inlier list (ascending row order) and fitting
    a model to those rows; such a model also replaces the best one on ties;
  * the stopping rule after every model: stop once log(0.01) / log(min(1 - eps, 1 - ratio^3)) < i, i the outer
    iteration; the result is the best model's `lo_model`, R = lo_model^T;
  * chord inliers ||R b2 - b1|| < threshold, and the pair's score: the outliers if they are at least 30 % of the
    rows, else 0.

The rotation of a sample (geometry::RotationBetweenPoints) is the orthogonal polar factor of the centred
cross-covariance M = sum (b1_i - mean b1) (b2_i - mean b2)^T, negated if improper.  A 3-row sample makes M rank 2, so
that rule is decided by round-off there; for exactly 3 rows the rotation is instead the proper (Kabsch) completion,
the polar factor of M + (|M| / |cof M|) cof M (cof M = sigma1 sigma2 (u1 x u2)(v1 x v2)^T for a rank-2 M).  Both are
computed by the same scaled Newton iteration as the device.  A sample whose matrix is singular gets the identity.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np

SEED = 42
PROBABILITY = 0.99
LO_ITERATIONS = 10
LO_SAMPLE_CLAMP = 12
MINIMAL_SAMPLES = 3
NEWTON_MAX_ITERATIONS = 50
NEWTON_UNSCALED_BELOW = 1e-2   # Frobenius step below which the Newton iteration stops scaling
NEWTON_TOLERANCE = 1e-14       # Frobenius step below which it stops
DBL_EPSILON = np.finfo(np.float64).eps

_M32 = 0xFFFFFFFF


class Mt19937:
    """std::mt19937: the 32-bit Mersenne twister (Matsumoto and Nishimura, 1998) with its standard seeding."""

    N, M = 624, 397

    def __init__(self, seed: int = 5489):
        s = np.zeros(self.N, dtype=np.uint64)
        s[0] = seed & _M32
        for k in range(1, self.N):
            p = int(s[k - 1])
            s[k] = (1812433253 * (p ^ (p >> 30)) + k) & _M32
        self.state = s.astype(np.uint32)
        self.index = self.N

    def _twist(self) -> None:
        s = self.state.astype(np.uint64)
        N, M = self.N, self.M
        for k in range(N):
            y = (int(s[k]) & 0x80000000) | (int(s[(k + 1) % N]) & 0x7FFFFFFF)
            v = int(s[(k + M) % N]) ^ (y >> 1)
            if y & 1:
                v ^= 0x9908B0DF
            s[k] = v
        self.state = s.astype(np.uint32)
        self.index = 0

    def outputs(self, count: int) -> np.ndarray:
        out = np.empty(count, dtype=np.uint32)
        for j in range(count):
            if self.index >= self.N:
                self._twist()
            y = int(self.state[self.index])
            self.index += 1
            y ^= y >> 11
            y ^= (y << 7) & 0x9D2C5680
            y ^= (y << 15) & 0xEFC60000
            y ^= y >> 18
            out[j] = y
        return out


class SampleStream:
    """The raw outputs of mt19937(42), shared by every pair: a cached prefix, extended on demand."""

    _cache = np.zeros(0, dtype=np.uint32)
    _gen: Optional[Mt19937] = None

    @classmethod
    def prefix(cls, count: int) -> np.ndarray:
        if len(cls._cache) < count:
            if cls._gen is None:
                cls._gen = Mt19937(SEED)
            more = max(count - len(cls._cache), 4096)
            cls._cache = np.concatenate([cls._cache, cls._gen.outputs(more)])
        return cls._cache

    def __init__(self):
        self.cursor = 0

    def next(self) -> int:
        if self.cursor >= len(SampleStream._cache):
            SampleStream.prefix(self.cursor + 1)
        v = int(SampleStream._cache[self.cursor])
        self.cursor += 1
        return v


def draw(stream: SampleStream, n: int) -> int:
    """uniform_int_distribution<unsigned long>(0, n - 1) over a 32-bit generator, libstdc++ 13: Lemire's 64-bit
    product, rejecting low words below 2^32 mod n."""
    product = stream.next() * n
    low = product & _M32
    if low < n:
        threshold = ((1 << 32) - n) % n
        while low < threshold:
            product = stream.next() * n
            low = product & _M32
    return product >> 32


def sample(stream: SampleStream, size: int, n: int) -> List[int]:
    """`size` distinct indices in [0, n), in draw order; a repeated index is drawn again."""
    out: List[int] = []
    for _ in range(size):
        v = draw(stream, n)
        while v in out:
            v = draw(stream, n)
        out.append(v)
    return out


# ---------------------------------------------------------------------------------------------------------------
# 3x3 algebra, written in the device's operation order
# ---------------------------------------------------------------------------------------------------------------
def cofactor(X: np.ndarray) -> np.ndarray:
    """Columns c1 x c2, c2 x c0, c0 x c1: X^T cof(X) = det(X) I."""
    c0, c1, c2 = X[:, 0], X[:, 1], X[:, 2]
    return np.column_stack([np.cross(c1, c2), np.cross(c2, c0), np.cross(c0, c1)])


def polar(X: np.ndarray) -> Optional[np.ndarray]:
    """Orthogonal polar factor by Newton's iteration X <- (z X + X^-T / z) / 2, with Frobenius-norm scaling z until
    the step falls below NEWTON_UNSCALED_BELOW; None if X is singular."""
    nx = float(np.sqrt(np.sum(X * X)))
    if not np.isfinite(nx) or nx == 0.0:
        return None
    X = X / nx
    scaled = True
    for _ in range(NEWTON_MAX_ITERATIONS):
        C = cofactor(X)
        d = float(np.dot(X[:, 0], C[:, 0]))
        if d == 0.0 or not np.isfinite(d):
            return None
        Y = C / d
        if scaled:
            z = float(np.sqrt(np.sqrt(np.sum(Y * Y)) / np.sqrt(np.sum(X * X))))
            Xn = 0.5 * (z * X + Y / z)
        else:
            Xn = 0.5 * (X + Y)
        step = float(np.sqrt(np.sum((Xn - X) ** 2)))
        X = Xn
        if step < NEWTON_UNSCALED_BELOW:
            scaled = False
        if step <= NEWTON_TOLERANCE:
            break
    return X if np.all(np.isfinite(X)) else None


def rotation_between(b1: np.ndarray, b2: np.ndarray) -> np.ndarray:
    """The rotation Q with Q b2 ~ b1 of the rows (in order): see the module docstring.  The model is Q^T."""
    k = len(b1)
    m1 = b1[0].copy()
    m2 = b2[0].copy()
    for i in range(1, k):
        m1 += b1[i]
        m2 += b2[i]
    m1 /= k
    m2 /= k
    M = np.zeros((3, 3))
    for i in range(k):
        M += np.outer(b1[i] - m1, b2[i] - m2)
    if k == MINIMAL_SAMPLES:
        C = cofactor(M)
        nc = float(np.sqrt(np.sum(C * C)))
        if nc > 0.0:
            M = M + (float(np.sqrt(np.sum(M * M))) / nc) * C
    Q = polar(M)
    if Q is None:
        return np.eye(3)
    if np.linalg.det(Q) < 0.0:
        Q = -Q
    return Q


def errors(model: np.ndarray, b1: np.ndarray, b2: np.ndarray) -> np.ndarray:
    """1 - (model b1_i) . b2_i."""
    v = b1 @ model.T
    return 1.0 - (v[:, 0] * b2[:, 0] + v[:, 1] * b2[:, 1] + v[:, 2] * b2[:, 2])


def chord(R: np.ndarray, b1: np.ndarray, b2: np.ndarray) -> np.ndarray:
    d = b2 @ R.T - b1
    return np.sqrt(d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2])


def stop_bound(inliers: int, n: int) -> float:
    """ShouldStop's iteration bound: stop once it is below the outer iteration index."""
    ratio = float(inliers) / n
    p = min(1.0 - DBL_EPSILON, 1.0 - ratio ** 3.0)
    return float(np.log(1.0 - PROBABILITY) / np.log(p)) if p > 0.0 else float(np.log(1.0 - PROBABILITY) / -np.inf)


@dataclass
class PairResult:
    lo_model: np.ndarray                 # 3x3; R = lo_model.T
    ransac_inliers: int
    chord_mask: np.ndarray               # bool per row
    chord_inliers: int
    score: int                           # pairwise_reconstructability
    draws: List[int] = field(default_factory=list)   # every accepted sample index, in order (LO: inlier-list positions)
    iterations: int = 0                  # outer iterations run
    stream_used: int = 0                 # raw generator outputs consumed
    error_margin: float = np.inf         # min | |e| - (1 - cos threshold) | over every model evaluated
    chord_margin: float = np.inf         # min | chord - threshold | of the final model
    stop_margin: float = np.inf          # min | bound - i | over every ShouldStop evaluation
    events: List[tuple] = field(default_factory=list)  # per outer iteration: (inliers, best before, replaced, LO ran)

    @property
    def R(self) -> np.ndarray:
        return self.lo_model.T


def reconstructability(common: int, rotation_inliers: int) -> int:
    """pairwise_reconstructability (an int: the reference returns the outlier count or 0)."""
    outliers = common - rotation_inliers
    return outliers if float(outliers) / common >= 0.3 else 0


def ransac_rotation(b1: np.ndarray, b2: np.ndarray, threshold: float, iterations: int = 1000) -> PairResult:
    b1 = np.ascontiguousarray(b1, dtype=np.float64).reshape(-1, 3)
    b2 = np.ascontiguousarray(b2, dtype=np.float64).reshape(-1, 3)
    n = len(b1)
    if n < MINIMAL_SAMPLES:
        raise ValueError("rotation RANSAC needs at least 3 correspondences, got %d" % n)
    t = 1.0 - np.cos(threshold)
    stream = SampleStream()
    res = PairResult(np.zeros((3, 3)), 0, np.zeros(n, bool), 0, 0)
    best_inliers = np.zeros(0, dtype=np.int64)
    best_lo = None

    def evaluate(model):
        e = np.abs(errors(model, b1, b2))
        res.error_margin = min(res.error_margin, float(np.min(np.abs(e - t))))
        return np.nonzero(e < t)[0]

    for i in range(iterations):
        idx = sample(stream, MINIMAL_SAMPLES, n)
        res.draws += idx
        model = rotation_between(b1[idx], b2[idx]).T
        inl = evaluate(model)
        res.iterations = i + 1
        replaced = len(inl) >= len(best_inliers)
        res.events.append((len(inl), len(best_inliers), replaced, replaced and len(inl) >= MINIMAL_SAMPLES))
        if replaced:
            best_inliers, best_lo = inl, model
            if len(inl) >= MINIMAL_SAMPLES:
                for _ in range(LO_ITERATIONS):
                    m = len(best_inliers)
                    size = max(min(LO_SAMPLE_CLAMP, int(m * 0.5)), MINIMAL_SAMPLES)
                    pos = sample(stream, size, m)
                    res.draws += pos
                    rows = best_inliers[pos]
                    lo = rotation_between(b1[rows], b2[rows]).T
                    lo_inl = evaluate(lo)
                    if len(lo_inl) >= len(best_inliers):
                        best_inliers, best_lo = lo_inl, lo
        bound = stop_bound(len(best_inliers), n)
        if len(best_inliers) < n:   # all rows inliers: the bound is exactly 0, not a rounding question
            res.stop_margin = min(res.stop_margin, abs(bound - i))
        if bound < i:
            break
    res.lo_model = best_lo
    res.ransac_inliers = len(best_inliers)
    c = chord(res.R, b1, b2)
    res.chord_margin = float(np.min(np.abs(c - threshold)))
    res.chord_mask = c < threshold
    res.chord_inliers = int(res.chord_mask.sum())
    res.score = reconstructability(n, res.chord_inliers)
    res.stream_used = stream.cursor
    return res
