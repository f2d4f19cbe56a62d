"""The deflation space of the reduced camera system (opensfm_b200/csrc/ba_reduced.cuh `pcg_gauge_vectors`, DESIGN.md (d)5):
the seven similarity-gauge directions of the rig instances.  CPU only: the formula is restated in numpy and checked
against the oracle's reduced system -- the directions are (near-)null vectors of S without damping, and projecting
them out of a block-Jacobi preconditioned CG cuts its iteration count, as it does for the CUDA solver."""
import numpy as np
import scipy.linalg as sl
from threadpoolctl import threadpool_limits

from opensfm_b200 import synthetic as syn
from oracle import ba_lm


def _gauge_vectors(inst, first_col, scale):
    """numpy restatement of pcg_gauge_vectors: instance block = [r (camera -> world angle-axis) | t (origin)];
    world map X -> s Q X + T moves t -> s Q t + T and R(r) -> Q R(r)."""
    n = len(scale)
    W = np.zeros((n, 7))
    for i, (r, t) in enumerate(zip(inst[:, :3], inst[:, 3:])):
        c0 = first_col + 6 * i
        th2 = r @ r
        g = 1.0 / 12.0
        if th2 > 1e-8:
            th = np.sqrt(th2)
            g = 1.0 / th2 - (1.0 + np.cos(th)) / (2.0 * th * np.sin(th))
        K = np.array([[0, -r[2], r[1]], [r[2], 0, -r[0]], [-r[1], r[0], 0]])
        Jl_inv = np.eye(3) - 0.5 * K + g * K @ K
        for a in range(3):
            e = np.zeros(3); e[a] = 1.0
            W[c0 + 3 + a, a] = 1.0                     # translation
            W[c0:c0 + 3, 3 + a] = Jl_inv[:, a]         # rotation: dr
            W[c0 + 3:c0 + 6, 3 + a] = np.cross(e, t)   # rotation: dt = e_a x t
        W[c0 + 3:c0 + 6, 6] = t                        # scale
    return W / scale[:, None]


def _pcg(S, b, blocks, W=None, tol=1e-8, maxit=5000):
    def M(r):
        z = np.empty_like(r)
        for idx, cf in blocks:
            z[idx] = sl.cho_solve(cf, r[idx])
        return z
    if W is not None:   # deflated CG (Saad, Yeung, Erhel, Guyomarc'h 2000)
        AW = S @ W
        cf = sl.cho_factor(W.T @ AW)
        x = W @ sl.cho_solve(cf, W.T @ b)
    else:
        x = np.zeros_like(b)
    r = b - S @ x
    z = M(r)
    p = z - W @ sl.cho_solve(cf, AW.T @ z) if W is not None else z.copy()
    rz, b2 = r @ z, b @ b
    for it in range(1, maxit + 1):
        Ap = S @ p
        a = rz / (p @ Ap)
        x += a * p
        r -= a * Ap
        if r @ r < tol * tol * b2:
            return it, x
        z = M(r)
        rz2 = r @ z
        p = z + (rz2 / rz) * p
        if W is not None:
            p -= W @ sl.cho_solve(cf, AW.T @ z)
        rz = rz2
    return maxit, x


def test_gauge_directions_are_the_weak_modes_and_deflating_them_pays():
    # The oracle's OpenMP reductions and the BLAS calls sum in an order that depends on the thread count, and where the
    # plain CG below crosses its stopping tolerance (hence its final error) is sensitive to that: one thread makes the
    # comparison reproducible.  The oracle library is loaded first so that the limit reaches its OpenMP runtime.
    ba_lm.lib()
    with threadpool_limits(1):
        _check_gauge_deflation()


def _check_gauge_deflation():
    sc = syn.cube_scene(24, 1500, 1.0, with_descriptors=False, max_obs_per_point=8)
    pb = syn.scene_to_problem(sc)
    ba = ba_lm.OracleBA(pb)
    ba.linearize()
    cn, _ = ba.colnorm_gradient()
    scale = 1.0 / (1.0 + np.sqrt(cn))
    ba.set_scale(scale)
    diag = np.clip(cn * scale * scale, 1e-6, 1e32)
    K = len(pb.cam_type)
    nc = ba.nc
    first_col = int(pb.cam_off[-1])   # reduced vector: [cameras | rig instances | ...], every block free here
    assert nc == first_col + 6 * len(pb.inst)
    W = _gauge_vectors(np.asarray(pb.inst), first_col, scale[:nc])
    # without damping the seven directions are null vectors of the reduced system (gauge freedom of a reconstruction
    # without GPS): Rayleigh quotients at round-off level against eigenvalues of order one
    S0, _ = ba.schur(np.zeros_like(diag))
    for a in range(7):
        v = W[:, a]
        # camera priors (focal, k1, k2) do not touch the poses: the gauge stays free
        assert abs(v @ S0 @ v) / (v @ v) < 1e-7, a
    # with the first LM damping (radius 1e4) they are the weak end of the spectrum, and deflation pays
    S, rhs = ba.schur(diag / 1e4)
    blocks = []
    for k in range(K):   # the engine's preconditioner groups: a camera and its rig instance
        c_lo, c_hi = int(pb.cam_off[k]), int(pb.cam_off[k + 1])
        idx = np.r_[c_lo:c_hi, first_col + 6 * k:first_col + 6 * k + 6]
        blocks.append((idx, sl.cho_factor(S[np.ix_(idx, idx)])))
    it_plain, x_plain = _pcg(S, rhs, blocks)
    it_defl, x_defl = _pcg(S, rhs, blocks, W)
    x_exact = sl.cho_solve(sl.cho_factor(S), rhs)
    assert it_defl < 0.75 * it_plain, (it_plain, it_defl)
    # both stop at |r| <= 1e-8 |b|; the deflated one is at least as close to the exact solution
    e_plain, e_defl = np.linalg.norm(x_plain - x_exact), np.linalg.norm(x_defl - x_exact)
    assert e_defl <= 1.5 * e_plain + 1e-12 * np.linalg.norm(x_exact)
