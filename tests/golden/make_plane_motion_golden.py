"""Make tests/golden/plane_motion_reference.npz: the first motion of OpenSfM's
`multiview.motion_from_plane_homography` on 52 homographies, so that opensfm_b200.relative_pose.plane_motions is
checked against it without the reference installed.

    python tests/golden/make_plane_motion_golden.py /path/to/OpenSfM

`import opensfm` needs its compiled modules, so the function alone is taken out of opensfm/multiview.py with `ast`
and run with numpy.  The fixture holds numbers only: H, and the reference's R and t of motion 0 (NaN when it
returns None).
"""
import ast
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))


def load_function(path: str, name: str):
    tree = ast.parse(open(path).read())
    node = next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == name)
    node.returns = None
    for a in node.args.args:
        a.annotation = None
    scope = {"np": np}
    exec(compile(ast.Module(body=[node], type_ignores=[]), path, "exec"), scope)
    return scope[name]


def homographies():
    """H = d R + t n^T of random motions and planes (40), the same with 1e-3 relative noise (10), and two with
    repeated singular values."""
    rng = np.random.RandomState(3)
    out = []
    for k in range(50):
        w = rng.randn(3) * rng.uniform(0.05, 0.6)
        th = np.linalg.norm(w)
        K = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]]) / th
        R = np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K
        t = rng.randn(3)
        n = rng.randn(3)
        n /= np.linalg.norm(n)
        H = rng.uniform(0.5, 5.0) * R + np.outer(t, n)
        if k >= 40:
            H = H + 1e-3 * np.abs(H).max() * rng.randn(3, 3)
        out.append(H * rng.uniform(0.2, 3.0))
    out.append(np.eye(3))
    out.append(np.diag([2.0, 2.0, 1.0]))
    return np.array(out)


def main():
    root = sys.argv[1]
    f = load_function(os.path.join(root, "opensfm", "multiview.py"), "motion_from_plane_homography")
    Hs = homographies()
    R = np.full((len(Hs), 3, 3), np.nan)
    t = np.full((len(Hs), 3), np.nan)
    for k, H in enumerate(Hs):
        m = f(H)
        if m:
            R[k], t[k] = m[0][0], m[0][1]
    np.savez_compressed(os.path.join(HERE, "plane_motion_reference.npz"), H=Hs, R=R, t=t)
    print("%d homographies, %d without motions" % (len(Hs), int(np.isnan(t[:, 0]).sum())))


if __name__ == "__main__":
    main()
