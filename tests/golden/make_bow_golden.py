"""Fixture of the BoW tests: a seeded 1024-word subset of the reference's 10000-word BoW vocabulary and its word
frequencies, made HERE from the reference's own vocabulary file, which is not part of this repository:

    python tests/golden/make_bow_golden.py OPENSFM_CHECKOUT   # reads opensfm/data/bow/bow_hahog_root_uchar_10000.npz in it

Saved as bow_words_1024.npz: `words` (1024 x 128 float32, rows of the vocabulary in ascending index order),
`frequencies` (their entries of the vocabulary's `frequencies`), `index` (the rows taken) and the seed."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
BOW_FILE = os.path.join("opensfm", "data", "bow", "bow_hahog_root_uchar_10000.npz")
SEED, NWORDS = 0, 1024

if __name__ == "__main__":
    bow = np.load(os.path.join(sys.argv[1], BOW_FILE))
    words, freq = bow["words"], bow["frequencies"]
    assert words.dtype == np.float32 and words.shape == (10000, 128), (words.dtype, words.shape)
    index = np.sort(np.random.RandomState(SEED).choice(len(words), NWORDS, replace=False))
    np.savez_compressed(os.path.join(HERE, "bow_words_1024.npz"), words=words[index], frequencies=freq[index],
                        index=index, seed=SEED)
    print("vocabulary", words.shape, freq.dtype, "integer-valued:", bool(np.all(words == np.round(words))),
          "zero frequencies:", int((freq == 0).sum()))
