"""Fixture of the VLAD tests: the reference's 64-word VLAD vocabulary, made HERE from the reference's own vocabulary
file, which is not part of this repository:

    python tests/golden/make_vlad_golden.py OPENSFM_CHECKOUT   # reads opensfm/data/bow/bow_hahog_root_uchar_64.npz in it

Saved: its `words` (64 x 128 float32, the centres `bow.load_vlad_words_and_frequencies` returns) as vlad_words_64.npz."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
VOCAB_FILE = os.path.join("opensfm", "data", "bow", "bow_hahog_root_uchar_64.npz")

if __name__ == "__main__":
    words = np.load(os.path.join(sys.argv[1], VOCAB_FILE))["words"]
    assert words.dtype == np.float32 and words.shape == (64, 128), (words.dtype, words.shape)
    np.savez_compressed(os.path.join(HERE, "vlad_words_64.npz"), words=words)
    print("vocabulary", words.shape, "integer-valued:", bool(np.all(words == np.round(words))))
