"""Generates tests/golden/resection_oracle.npz: oracle/absolute_pose_oracle.py on every shot of the batch
tests/test_resection_gpu.py compares the engine with (resection_cases.batch_shots(), regenerated from its seed).  The
oracle runs local optimisation's Lu iterations in Python and takes tens of CPU-minutes on the batch, so its results
are kept here rather than recomputed on every GPU run.

    python tests/golden/make_resection_golden.py
"""
import multiprocessing
import os
import sys
from concurrent.futures import ProcessPoolExecutor

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
sys.path.insert(0, os.path.join(HERE, ".."))
import resection_cases as C  # noqa: E402
from oracle import absolute_pose_oracle as o  # noqa: E402

OUT = os.path.join(HERE, "resection_oracle.npz")


def main():
    bs, Xs = C.batch_shots()
    order = sorted(range(len(bs)), key=lambda k: -len(bs[k]))
    with ProcessPoolExecutor(os.cpu_count() or 1, mp_context=multiprocessing.get_context("spawn")) as ex:
        futures = {k: ex.submit(o.ransac_absolute_pose, bs[k], Xs[k], C.THRESHOLD) for k in order}
        res = [futures[k].result() for k in range(len(bs))]
    draws = [np.asarray(r.draws, dtype=np.int16) for r in res]
    np.savez_compressed(
        OUT,
        inputs_digest=np.array(C.digest(bs, Xs)),
        draw_start=np.concatenate([[0], np.cumsum([len(d) for d in draws])]).astype(np.int64),
        draws=np.concatenate(draws),
        stream_used=np.array([r.stream_used for r in res], dtype=np.int64),
        ransac_inliers=np.array([r.ransac_inliers for r in res], dtype=np.int32),
        chord_inliers=np.array([r.chord_inliers for r in res], dtype=np.int32),
        chord_mask=np.packbits(np.concatenate([r.chord_mask for r in res])),
        lo_model=np.array([r.lo_model for r in res]),
        margins=np.array([[r.error_margin, r.chord_margin, r.stop_margin, r.lu_margin] for r in res]))
    print(OUT)


if __name__ == "__main__":
    main()
