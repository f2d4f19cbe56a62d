"""Writes tests/golden/relative_pose_oracle.npz: oracle/relative_pose_oracle.py's result on every pair of
relative_pose_cases.batch_pairs(), which takes CPU-minutes.  Run from the repository root:

    python tests/golden/make_relative_pose_golden.py
"""
import os
import sys
from multiprocessing import Pool

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

import relative_pose_cases as C  # noqa: E402
from oracle import relative_pose_oracle as ro  # noqa: E402


def one(args):
    b1, b2 = args
    r = ro.ransac_relative_pose(b1, b2, C.THRESHOLD)
    return (np.array(r.draws, np.int32), r.stream_used, r.ransac_inliers, r.inlier_mask, r.lo_model,
            np.array([r.error_margin, r.stop_margin, r.class_margin, r.decomposition_margin, r.ratio_margin]))


def main():
    b1s, b2s = C.batch_pairs()
    with Pool() as pool:
        out = pool.map(one, list(zip(b1s, b2s)), chunksize=1)
    draws = [o[0] for o in out]
    draw_start = np.concatenate([[0], np.cumsum([len(d) for d in draws])]).astype(np.int64)
    np.savez_compressed(os.path.join(HERE, "relative_pose_oracle.npz"),
                        inputs_digest=C.digest(b1s, b2s),
                        draws=np.concatenate(draws), draw_start=draw_start,
                        stream_used=np.array([o[1] for o in out], np.int64),
                        ransac_inliers=np.array([o[2] for o in out], np.int32),
                        inlier_mask=np.packbits(np.concatenate([o[3] for o in out])),
                        lo_model=np.array([o[4] for o in out]),
                        margins=np.array([o[5] for o in out]))


if __name__ == "__main__":
    main()
