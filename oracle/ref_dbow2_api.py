"""ctypes wrapper of oracle/_ref/libdbow2_ref.so: the REFERENCE's own DBoW2 (ThirdParty/DBoW2) compiled in place by
`make -C oracle ref`.  TEST INFRASTRUCTURE: pins oracle/mcs_oracle.cpp's bag-of-words restatement and generates
tests/golden/bow_small_voc.npz (tests/golden/make_bow_golden.py)."""
import ctypes as C
import pathlib

import numpy as np

_HERE = pathlib.Path(__file__).resolve().parent
SO = _HERE / "_ref" / "libdbow2_ref.so"
VOC_TXT = _HERE / "_ref" / "voc_small_9_6.txt"


def available():
    return SO.exists() and VOC_TXT.exists()


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


class RefVocabulary:
    def __init__(self, txt=VOC_TXT, scoring=None, weighting=None):
        self.lib = C.CDLL(str(SO))
        self.lib.refbow_load_text.restype = C.c_void_p
        self.lib.refbow_score.restype = C.c_double
        self.h = C.c_void_p(self.lib.refbow_load_text(str(txt).encode()))
        if not self.h:
            raise RuntimeError("reference vocabulary did not load")
        if scoring is not None or weighting is not None:
            self.set_types(scoring, weighting)

    def set_types(self, scoring, weighting):
        """the scoring and weighting types, without loading the tree again"""
        self.lib.refbow_set_types(self.h, int(scoring), int(weighting))

    def __del__(self):
        if getattr(self, "h", None):
            self.lib.refbow_free(self.h); self.h = None

    def size(self):
        return self.lib.refbow_size(self.h)

    def transform(self, desc, levelsup=4):
        desc = np.ascontiguousarray(desc, np.uint8); n = len(desc)
        bw = np.zeros(max(n, 1), np.int32); bv = np.zeros(max(n, 1), np.float64); nb = C.c_int(0)
        fn = np.zeros(max(n, 1), np.int32); fo = np.zeros(n + 2, np.int32); nf = C.c_int(0); ff = np.zeros(max(n, 1), np.int32)
        self.lib.refbow_transform(self.h, _p(desc), n, levelsup, _p(bw), _p(bv), C.byref(nb), _p(fn), _p(fo), C.byref(nf), _p(ff))
        return bw[:nb.value].copy(), bv[:nb.value].copy(), fn[:nf.value].copy(), fo[:nf.value + 1].copy(), ff[:fo[nf.value]].copy()

    def words(self, desc):
        desc = np.ascontiguousarray(desc, np.uint8); n = len(desc)
        w = np.zeros(n, np.int32); wt = np.zeros(n, np.float64)
        self.lib.refbow_words(self.h, _p(desc), n, _p(w), _p(wt))
        return w, wt

    def score(self, w1, v1, w2, v2):
        w1 = np.ascontiguousarray(w1, np.int32); w2 = np.ascontiguousarray(w2, np.int32)
        v1 = np.ascontiguousarray(v1, np.float64); v2 = np.ascontiguousarray(v2, np.float64)
        return self.lib.refbow_score(self.h, _p(w1), _p(v1), len(w1), _p(w2), _p(v2), len(w2))
