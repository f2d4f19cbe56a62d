"""Track creation restated for the tests -- test infrastructure only.

What `tracking.create_tracks_manager` computes (opensfm/tracking.py:72-150, 238-244) and what the reconstruction
then asks of the result for every image pair (tracks_manager.cc:285-350), written from that behaviour with an
algorithm that shares nothing with the engine's:

  * the features that occur in a match are the nodes, the match rows the edges; tracks are the connected
    components (`scipy.sparse.csgraph.connected_components`);
  * a component is kept if it has at least `min_length` features and no two of one image -- counted over all its
    features, also those of images without a feature file;
  * features of images without a feature file are then left out; a track with nothing left does not exist;
  * two images have a track in common when both observe it.

`tracks(...)` returns the partition as a set of frozensets of (image, feature) and
{(im1, im2): [(feature1, feature2), ...]} with im1 < im2, one entry per common track.
"""
from __future__ import annotations

from typing import Any, Dict, FrozenSet, Iterable, List, Set, Tuple

import numpy as np
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components


def tracks(images_with_features: Iterable[Any], matches: Dict[Tuple[Any, Any], Any], min_length: int,
           with_common: bool = True
           ) -> Tuple[Set[FrozenSet[Tuple[Any, int]]], Dict[Tuple[Any, Any], List[Tuple[int, int]]]]:
    """with_common=False leaves the second result empty (its loop is quadratic in a track's length)."""
    with_features = set(images_with_features)
    names = sorted({im for pair in matches for im in pair})
    index = {im: i for i, im in enumerate(names)}
    rows = [np.asarray(m, dtype=np.int64).reshape(-1, 2) for m in matches.values()]
    if not rows or not sum(len(r) for r in rows):
        return set(), {}
    span = max(int(r.max()) for r in rows if len(r)) + 1
    # node key = image * span + feature; compact ids through np.unique
    ka = np.concatenate([index[a] * span + r[:, 0] for (a, _), r in zip(matches, rows)])
    kb = np.concatenate([index[b] * span + r[:, 1] for (_, b), r in zip(matches, rows)])
    keys, inv = np.unique(np.concatenate([ka, kb]), return_inverse=True)
    u, v = inv[:len(ka)], inv[len(ka):]
    n = len(keys)
    graph = coo_matrix((np.ones(len(u), dtype=np.int8), (u, v)), shape=(n, n))
    _, label = connected_components(graph, directed=False)
    order = np.argsort(label, kind="stable")
    bounds = np.flatnonzero(np.diff(label[order])) + 1
    partition: Set[FrozenSet[Tuple[Any, int]]] = set()
    common: Dict[Tuple[Any, Any], List[Tuple[int, int]]] = {}
    for comp in np.split(order, bounds):
        img = keys[comp] // span
        if len(comp) < min_length or len(np.unique(img)) != len(img):
            continue
        obs = sorted((names[i], int(k % span)) for i, k in zip(img.tolist(), keys[comp].tolist())
                     if names[i] in with_features)
        if not obs:
            continue
        partition.add(frozenset(obs))
        for x in range(len(obs) if with_common else 0):
            for y in range(x + 1, len(obs)):
                common.setdefault((obs[x][0], obs[y][0]), []).append((obs[x][1], obs[y][1]))
    return partition, common
