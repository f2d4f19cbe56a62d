"""Five-point relative-pose RANSAC of one image pair in numpy: the CPU restatement that opensfm_b200/csrc/relpose.cu
(and the solvers of opensfm_b200/csrc/relative_pose.cuh) are checked against.

What it restates: pyrobust's `ransac_relative_pose` with RANSAC scoring as `multiview.relative_pose_ransac` calls it
(only `iterations` is set, so the stopping rule uses probability 0.99):

  * rows: a pair of bearings (x in the first image, y in the second), normalised once;
  * the sample stream and the draws of the rotation RANSAC (rotation_ransac_oracle): mt19937(42) restarted for
    every pair, 5-row samples; the stopping bound log(0.01) / log(min(1 - eps, 1 - ratio^5));
  * the models of a sample: EssentialFivePoints (geometry/essential.h) -- the nullspace of the 5 epipolar rows, the
    10 x 20 constraint matrix (det E = 0, 2 E E^T E - tr(E E^T) E = 0), Gauss-Jordan without pivoting (no model on a
    zero diagonal), the action matrix of multiplication by x, one essential per real eigenvalue from its
    eigenvector (x, y, z = v6 / v9, v7 / v9, v8 / v9), normalised -- each decomposed by RelativePoseFromEssential:
    t = +-u3, R = U W V^T or U W^T V^T with det U = det V = 1, the candidate of largest score on the sample rows
    (the sum of (px . x + py . y) / 2 over the rows whose midpoint triangulation has |det| >= 1e-10), the first of
    equal ones, when it scores above 0 (see below for the reference's int-kept score);
  * the error 1 - (px . x + py . y) / 2 of the midpoint of the row under [R | t] (1 when |det| < 1e-10), an
    inlier when its absolute value is below 1 - cos(threshold);
  * the model loop of robust_estimator.h: models scored in order, a model replaces the best one when it has at least
    as many inliers; whenever one does with at least 5 inliers, 10 rounds of local optimisation, each drawing
    max(min(12, floor(inliers / 2)), 5) positions of the best inlier list (ascending rows) and fitting
    EssentialNPoints (no model below 9 rows, nor when sigma_8 / sigma_9 <= 4; else the smallest right singular
    vector projected onto singular values ((a + b) / 2, (a + b) / 2, 0)), decomposed on the LO rows; the stopping
    rule after every model with the outer iteration index;
  * the result: the best model's lo_model [R | t] (x2 = R x1 + t) and the inlier mask of lo_model.

Deliberate differences from pyrobust, shared with the engine:
  * Eigen's EigenSolver returns the action matrix's eigenvalues in an order that depends on its QR iteration, which
    no device code can replay.  The real essentials of a sample are put in a canonical order instead: ascending
    eigenvalue.  The order only matters for exact ties between models of one sample;
  * the reference keeps a solution when its essential has an imaginary part of exactly zero, which is decided by
    round-off for close eigenvalues.  Here an eigenvalue is real when |Im| <= 1e-6 (1 + |Re|); the margin of that
    rule is recorded (`class_margin`);
  * JacobiSVD is replaced by eigen-decompositions of symmetric products: the nullspace of the five-point system by
    Householder QR of its transpose, the singular values of the N-point system by the eigenvalues of A^T A, and E's
    singular vectors by those of E^T E (u_k = E v_k / |E v_k|, u3 = u1 x u2, v3 = v1 x v2);
  * the choice among the four decompositions.  The reference keeps its best score in an int
    (std::pair<int, Matrix>, geometry/relative_pose.h:36, 73-77): a candidate wins when its score exceeds the best
    score so far truncated toward zero, so a later 1.2 beats an earlier 1.4.  That rule cannot be replayed: the
    candidates' order follows the signs Eigen's JacobiSVD gives E's singular vectors, and on rows an essential fits
    exactly (every five-point sample) each score sits at an integer -- each row agrees by +1, -1 or 0 -- where the
    comparison and the truncation are decided by round-off (a winner at 0.9999999999999998 keeps 0, and a later
    candidate at +1e-17 replaces it).  Here the candidate of largest score wins, which is what the reference's rule
    picks whenever the winner is not decided by round-off or by the order; the gap between the winning score and
    every other candidate's (and 0) is recorded (`decomposition_margin`);
  * when no decomposition scores above 0 the reference returns an uninitialised matrix; here it is all zeros, a pose
    under which no row triangulates;
  * rows come in the order the caller gives them, and a bearing is normalised once.

The engine's eigenvalues come from its own Hessenberg QR, the oracle's from LAPACK (numpy.linalg.eigvals), and the
oracle's symmetric eigen-decompositions from numpy.linalg.eigh: the comparison is also a check of the device's
linear algebra, at the cost of last-bit differences that the recorded margins bound.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional, Tuple

import numpy as np

from .rotation_ransac_oracle import DBL_EPSILON, LO_ITERATIONS, LO_SAMPLE_CLAMP, PROBABILITY, SampleStream, sample

MINIMAL_SAMPLES = 5
MIDPOINT_DET_EPS = 1e-10
REAL_TOLERANCE = 1e-6
NULLSPACE_RATIO = 4.0


# ---------------------------------------------------------------------------------------------------------------
# polynomials in x, y, z of degree <= 3, in the reference's monomial order
# ---------------------------------------------------------------------------------------------------------------
def _monomials() -> List[Tuple[int, int, int]]:
    """(x, y, z) exponents: by degree descending, then by the power of z, then by the power of y."""
    out = []
    for d in (3, 2, 1, 0):
        for ez in range(d + 1):
            for ey in range(d - ez + 1):
                out.append((d - ey - ez, ey, ez))
    return out


MONOMIALS = _monomials()
_INDEX = {m: k for k, m in enumerate(MONOMIALS)}


def _product_table(first_a: int, first_b: int):
    ii, jj, kk = [], [], []
    for i in range(first_a, 20):
        for j in range(first_b, 20):
            m = tuple(p + q for p, q in zip(MONOMIALS[i], MONOMIALS[j]))
            ii.append(i)
            jj.append(j)
            kk.append(_INDEX[m])
    return np.array(ii), np.array(jj), np.array(kk)


_LIN_LIN = _product_table(16, 16)
_QUAD_LIN = _product_table(10, 16)


def poly_mul(a: np.ndarray, b: np.ndarray, quad: bool) -> np.ndarray:
    """a * b for a linear (or, `quad`, quadratic) a and a linear b."""
    i, j, k = _QUAD_LIN if quad else _LIN_LIN
    out = np.zeros(20)
    np.add.at(out, k, a[i] * b[j])
    return out


# ---------------------------------------------------------------------------------------------------------------
# the five-point solver
# ---------------------------------------------------------------------------------------------------------------
def epipolar_rows(x1: np.ndarray, x2: np.ndarray) -> np.ndarray:
    """Rows of x2^T E x1 = 0 in E's row-major entries."""
    return np.einsum("ki,kj->kij", x2, x1).reshape(-1, 9)


def nullspace5(x1: np.ndarray, x2: np.ndarray) -> np.ndarray:
    """9 x 4: the last 4 columns of Q of the Householder QR of A^T, A the 5 x 9 epipolar system."""
    W = epipolar_rows(x1, x2).T.copy()
    vs, betas = [], []
    for j in range(5):
        nx = float(np.sqrt(np.sum(W[j:, j] ** 2)))
        alpha = -nx if W[j, j] >= 0.0 else nx
        v = np.zeros(9)
        v[j:] = W[j:, j]
        v[j] -= alpha
        beta = float(v @ v)
        vs.append(v)
        betas.append(beta)
        if beta != 0.0:
            W -= np.outer(v, 2.0 * (v @ W) / beta)
    N = np.zeros((9, 4))
    for c in range(4):
        e = np.zeros(9)
        e[5 + c] = 1.0
        for j in range(4, -1, -1):
            if betas[j] != 0.0:
                e -= (2.0 * float(vs[j] @ e) / betas[j]) * vs[j]
        N[:, c] = e
    return N


def constraints(N: np.ndarray) -> np.ndarray:
    """The 10 x 20 constraint matrix: det E, then the rows of (E E^T - tr(E E^T) / 2 I) E, row-major."""
    E = np.zeros((9, 20))
    E[:, 16:20] = N
    M = np.zeros((10, 20))
    for j in range(3):
        j1, j2 = (j + 1) % 3, (j + 2) % 3
        minor = poly_mul(E[3 + j1], E[6 + j2], False) - poly_mul(E[3 + j2], E[6 + j1], False)
        M[0] += poly_mul(minor, E[j], True)
    L = np.zeros((9, 20))
    for i in range(3):
        for j in range(i, 3):
            L[3 * i + j] = sum(poly_mul(E[3 * i + k], E[3 * j + k], False) for k in range(3))
            L[3 * j + i] = L[3 * i + j]
    half_trace = 0.5 * (L[0] + L[4] + L[8])
    for i in range(3):
        L[4 * i] -= half_trace
    for i in range(3):
        for j in range(3):
            M[1 + 3 * i + j] = sum(poly_mul(L[3 * i + k], E[3 * k + j], True) for k in range(3))
    return M


def gauss_jordan(M: np.ndarray) -> bool:
    """FivePointsGaussJordan, in place: each row divided by its diagonal, row_j <- row_j / M[j, i] - row_i below
    (skipped when M[j, i] is 0), then back-substitution; False on a zero diagonal."""
    for i in range(10):
        d = M[i, i]
        if d == 0.0:
            return False
        M[i] /= d
        for j in range(i + 1, 10):
            e = M[j, i]
            if e != 0.0:
                M[j] = M[j] / e - M[i]
    for i in range(9, -1, -1):
        for j in range(i):
            M[j] -= M[j, i] * M[i]
    return True


def action_matrix(M: np.ndarray) -> np.ndarray:
    A = np.zeros((10, 10))
    A[:6] = -M[[0, 1, 2, 4, 5, 7], 10:]
    A[6, 0] = A[7, 1] = A[8, 3] = A[9, 6] = 1.0
    return A


def null_vector10(B: np.ndarray) -> np.ndarray:
    """A null vector of B by Gaussian elimination with complete pivoting; the last unknown is 1 (0 for a zero
    pivot)."""
    B = B.copy()
    col = list(range(10))
    for k in range(9):
        sub = np.abs(B[k:, k:])
        flat = int(np.argmax(sub))
        pi, pj = k + flat // (10 - k), k + flat % (10 - k)
        B[[k, pi]] = B[[pi, k]]
        B[:, [k, pj]] = B[:, [pj, k]]
        col[k], col[pj] = col[pj], col[k]
        d = B[k, k]
        if d == 0.0:
            continue
        f = B[k + 1:, k] / d
        B[k + 1:, k:] -= np.outer(f, B[k, k:])
    y = np.zeros(10)
    y[9] = 1.0
    for k in range(8, -1, -1):
        s = float(B[k, k + 1:] @ y[k + 1:])
        y[k] = 0.0 if B[k, k] == 0.0 else -s / B[k, k]
    v = np.zeros(10)
    v[col] = y
    return v


def real_eigenvalues(A: np.ndarray) -> Tuple[List[float], float]:
    """(the real eigenvalues of A ascending, the classification margin); LAPACK's eigenvalues."""
    w = np.linalg.eigvals(A)
    scale = 1.0 + np.abs(w.real)
    margin = np.inf
    nz = w.imag != 0.0
    if nz.any():
        margin = float(np.min(np.abs(np.abs(w.imag[nz]) - REAL_TOLERANCE * scale[nz]) / scale[nz]))
    real = np.abs(w.imag) <= REAL_TOLERANCE * scale
    return sorted(w.real[real].tolist()), margin


def five_point(x1: np.ndarray, x2: np.ndarray, margins: Optional[dict] = None) -> List[np.ndarray]:
    """EssentialFivePoints of 5 rows: the real essentials (3 x 3, unit Frobenius norm), by ascending eigenvalue."""
    N = nullspace5(x1, x2)
    M = constraints(N)
    if not gauss_jordan(M):
        return []
    A = action_matrix(M)
    if not np.all(np.isfinite(A)):
        return []
    roots, margin = real_eigenvalues(A)
    if margins is not None:
        margins["class"] = min(margins.get("class", np.inf), margin)
    out = []
    for lam in roots:
        v = null_vector10(A - lam * np.eye(10))
        with np.errstate(divide="ignore", invalid="ignore"):
            x, y, z = v[6] / v[9], v[7] / v[9], v[8] / v[9]
            E = x * N[:, 0] + y * N[:, 1] + z * N[:, 2] + N[:, 3]
            E = E / np.sqrt(E @ E)
        out.append(E.reshape(3, 3))
    return out


# ---------------------------------------------------------------------------------------------------------------
# N points, decomposition, error
# ---------------------------------------------------------------------------------------------------------------
def sym_eig(S: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """(eigenvalues descending, eigenvectors as columns) of a symmetric matrix."""
    w, V = np.linalg.eigh(S)
    return w[::-1], V[:, ::-1]


def essential_svd(E: np.ndarray):
    """(U, V, s) with u_k = E v_k / |E v_k| (k = 1, 2; u2 orthogonalised), u3 = u1 x u2, v3 = v1 x v2."""
    w, V = sym_eig(E.T @ E)
    u0 = E @ V[:, 0]
    u0 = u0 / np.sqrt(u0 @ u0)
    u1 = E @ V[:, 1]
    u1 = u1 - (u0 @ u1) * u0
    u1 = u1 / np.sqrt(u1 @ u1)
    U = np.column_stack([u0, u1, np.cross(u0, u1)])
    V = np.column_stack([V[:, 0], V[:, 1], np.cross(V[:, 0], V[:, 1])])
    return U, V, np.sqrt(np.maximum(w, 0.0))


def agreement(M: np.ndarray, x: np.ndarray, y: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """((px . x + py . y) / 2, whether the row triangulates) of every row under the pose M = [R | t]."""
    R, t = M[:, :3], M[:, 3]
    c1 = -(R.T @ t)
    by = y @ R
    r0, r1 = x @ c1, by @ c1
    a00 = np.einsum("ij,ij->i", x, x)
    a10 = np.einsum("ij,ij->i", x, by)
    a01, a11 = -a10, -np.einsum("ij,ij->i", by, by)
    det = a00 * a11 - a01 * a10
    ok = ~((-MIDPOINT_DET_EPS < det) & (det < MIDPOINT_DET_EPS))
    with np.errstate(divide="ignore", invalid="ignore"):
        l0 = (a11 * r0 - a01 * r1) / det
        l1 = (a00 * r1 - a10 * r0) / det
        X = 0.5 * (l0[:, None] * x + (c1[None, :] + l1[:, None] * by))
        px = X / np.sqrt(np.einsum("ij,ij->i", X, X))[:, None]
        Y = X @ R.T + t
        py = Y / np.sqrt(np.einsum("ij,ij->i", Y, Y))[:, None]
        a = (np.einsum("ij,ij->i", px, x) + np.einsum("ij,ij->i", py, y)) * 0.5
    return a, ok


def errors(M: np.ndarray, x: np.ndarray, y: np.ndarray) -> np.ndarray:
    """RelativePose::Evaluate of every row: 1 - agreement, 1 where the row does not triangulate."""
    a, ok = agreement(M, x, y)
    return np.where(ok, 1.0 - a, 1.0)


def decompositions(E: np.ndarray, x1: np.ndarray, x2: np.ndarray):
    """(the 4 candidate poses [R | t] of E: t = +u3, -u3 (outer), R = U W V^T, U W^T V^T (inner); their scores on
    the rows, the sum of agreement over the rows that triangulate)."""
    U, V, _ = essential_svd(E)
    poses, scores = [], []
    for i in range(2):
        t = U[:, 2] if i == 0 else -U[:, 2]
        t = t / np.sqrt(t @ t)
        for j in range(2):
            sg = 1.0 if j == 0 else -1.0
            R = sg * (np.outer(U[:, 1], V[:, 0]) - np.outer(U[:, 0], V[:, 1])) + np.outer(U[:, 2], V[:, 2])
            M = np.column_stack([R, t])
            with np.errstate(invalid="ignore"):
                a, ok = agreement(M, x1, x2)
                scores.append(float(np.sum(a[ok])))
            poses.append(M)
    return poses, scores


def pose_from_essential(E: np.ndarray, x1: np.ndarray, x2: np.ndarray,
                        margins: Optional[dict] = None) -> np.ndarray:
    """RelativePoseFromEssential scored on the rows (x1, x2): the candidate of largest score, the first of equal
    ones, above 0 ([R | t], 3 x 4), zeros when nothing scores above 0.  The reference keeps its best score in an
    int instead; see the module docstring for why that rule is not restated."""
    poses, scores = decompositions(E, x1, x2)
    best, win, out = 0.0, 4, np.zeros((3, 4))
    for c, (M, score) in enumerate(zip(poses, scores)):
        if score > best:
            best, win, out = score, c, M
    if margins is not None:
        gap = min(abs(best - s) for c, s in enumerate(scores + [0.0]) if c != win)
        margins["decomposition"] = min(margins.get("decomposition", np.inf), gap)
    return out


def n_points(x1: np.ndarray, x2: np.ndarray, margins: Optional[dict] = None) -> Optional[np.ndarray]:
    """EssentialNPoints: the essential of k >= 9 rows, or None."""
    if len(x1) < 9:
        return None
    A = epipolar_rows(x1, x2)
    w, V = sym_eig(A.T @ A)
    s7, s8 = np.sqrt(max(w[7], 0.0)), np.sqrt(max(w[8], 0.0))
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = s7 / s8
    if margins is not None:
        margins["ratio"] = min(margins.get("ratio", np.inf), abs(ratio - NULLSPACE_RATIO))
    if not ratio > NULLSPACE_RATIO:
        return None
    E0 = V[:, 8].reshape(3, 3)
    U, VE, s = essential_svd(E0)
    m = 0.5 * (s[0] + s[1])
    return m * (np.outer(U[:, 0], VE[:, 0]) + np.outer(U[:, 1], VE[:, 1]))


def stop_bound(inliers: int, n: int) -> float:
    """ShouldStop's iteration bound for 5-row samples."""
    ratio = float(inliers) / n
    p = min(1.0 - DBL_EPSILON, 1.0 - ratio ** 5.0)
    return float(np.log(1.0 - PROBABILITY) / np.log(p)) if p > 0.0 else float(np.log(1.0 - PROBABILITY) / -np.inf)


# ---------------------------------------------------------------------------------------------------------------
# the estimator
# ---------------------------------------------------------------------------------------------------------------
@dataclass
class PairResult:
    lo_model: np.ndarray                 # 3 x 4 [R | t], x2 = R x1 + t
    ransac_inliers: int
    inlier_mask: np.ndarray              # bool per row
    draws: List[int] = field(default_factory=list)   # every drawn sample index (LO: inlier-list positions)
    iterations: int = 0                  # outer iterations run
    stream_used: int = 0                 # raw generator outputs consumed
    error_margin: float = np.inf         # min | |e| - (1 - cos threshold) | over every model evaluated
    stop_margin: float = np.inf          # min | bound - i | over every ShouldStop evaluation
    class_margin: float = np.inf         # min relative distance of an eigenvalue's |Im| from the real-root rule
    decomposition_margin: float = np.inf  # min gap between a decomposition's winning score and another candidate's
    ratio_margin: float = np.inf         # min | sigma_8 / sigma_9 - 4 | of EssentialNPoints

    def pose(self) -> np.ndarray:
        """multiview.relative_pose_ransac's [R^T | -R^T t]."""
        R, t = self.lo_model[:, :3], self.lo_model[:, 3]
        return np.column_stack([R.T, -(R.T @ t)])


def normalize_rows(b: np.ndarray) -> np.ndarray:
    b = np.asarray(b, dtype=np.float64).reshape(-1, 3)
    return b / np.sqrt(b[:, 0] * b[:, 0] + b[:, 1] * b[:, 1] + b[:, 2] * b[:, 2])[:, None]


def sample_models(x1: np.ndarray, x2: np.ndarray, margins: Optional[dict] = None) -> List[np.ndarray]:
    """RelativePose::Estimate of a 5-row sample."""
    return [pose_from_essential(E, x1, x2, margins) for E in five_point(x1, x2, margins)]


def ransac_relative_pose(b1: np.ndarray, b2: np.ndarray, threshold: float, iterations: int = 1000) -> PairResult:
    x = normalize_rows(b1)
    y = normalize_rows(b2)
    n = len(x)
    if n < MINIMAL_SAMPLES or len(y) != n:
        raise ValueError("relative pose RANSAC needs at least 5 pairs of bearings, got %d" % n)
    t_err = 1.0 - np.cos(threshold)
    stream = SampleStream()
    res = PairResult(np.zeros((3, 4)), 0, np.zeros(n, bool))
    best_inliers = np.zeros(0, dtype=np.int64)
    best = np.zeros((3, 4))
    margins: dict = {}

    def evaluate(model):
        e = np.abs(errors(model, x, y))
        finite = np.isfinite(e)
        if finite.any():
            res.error_margin = min(res.error_margin, float(np.min(np.abs(e[finite] - t_err))))
        with np.errstate(invalid="ignore"):
            return np.nonzero(e < t_err)[0]

    stop = False
    for i in range(iterations):
        idx = sample(stream, MINIMAL_SAMPLES, n)
        res.draws += idx
        res.iterations = i + 1
        for model in sample_models(x[idx], y[idx], margins):
            inl = evaluate(model)
            if len(inl) >= len(best_inliers):
                best_inliers, best = inl, model
                if len(inl) >= MINIMAL_SAMPLES:
                    for _ in range(LO_ITERATIONS):
                        m = len(best_inliers)
                        size = max(min(LO_SAMPLE_CLAMP, int(m * 0.5)), MINIMAL_SAMPLES)
                        pos = sample(stream, size, m)
                        res.draws += pos
                        rows = best_inliers[pos]
                        E = n_points(x[rows], y[rows], margins)
                        if E is None:
                            continue
                        lo = pose_from_essential(E, x[rows], y[rows], margins)
                        lo_inl = evaluate(lo)
                        if len(lo_inl) >= len(best_inliers):
                            best_inliers, best = lo_inl, lo
            bound = stop_bound(len(best_inliers), n)
            if len(best_inliers) < n:   # all rows inliers: the bound is exactly 0, not a rounding question
                res.stop_margin = min(res.stop_margin, abs(bound - i))
            if bound < i:
                stop = True
                break
        if stop:
            break
    res.lo_model = best
    res.ransac_inliers = len(best_inliers)
    res.inlier_mask = np.zeros(n, bool)
    res.inlier_mask[best_inliers] = True
    res.stream_used = stream.cursor
    res.class_margin = margins.get("class", np.inf)
    res.decomposition_margin = margins.get("decomposition", np.inf)
    res.ratio_margin = margins.get("ratio", np.inf)
    return res
