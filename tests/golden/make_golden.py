"""Generates tests/golden/*.npz from oracle/_ref (`make -C oracle REF=<reference checkout>`):

    python tests/golden/make_golden.py

For every case in tests/cases.py it stores the SHA-256 of the raw I/Q bytes fed in and the outputs of
oracle/_ref/libairband_ref.so — i.e. the reference's OWN squelch.cpp / ctcss.cpp / filters.cpp (compiled in place
by oracle/Makefile) behind the restated demodulate() loop and the FP32 FFT stand-in, and in ref_leaf.npz the SHA-256
of the reference leaf classes' outputs that test_oracle_leaf_vs_ref.py and test_oracle_scan.py compare with."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle"), os.path.join(ROOT, "rtlsdr-airband_b200", "py")):
    sys.path.insert(0, p)

import hashlib  # noqa: E402

import oracle_py as op  # noqa: E402
from cases import CASES  # noqa: E402

GOLDEN = list(CASES)


def sha256(a: np.ndarray) -> np.ndarray:
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


def main():
    assert op.available("ref"), "build oracle/_ref first (make -C oracle)"
    for name in GOLDEN:
        cfg, raws = CASES[name]()
        res, o = op.run_oracle(cfg, raws, "ref")
        out = {}
        for d, (wo, iq, ax) in enumerate(res):
            out[f"raw{d}_sha256"] = sha256(raws[d])
            out[f"waveout{d}"] = wo
            out[f"iq_out{d}"] = iq
            out[f"axc{d}"] = ax
            st = []
            for c in range(wo.shape[0]):
                s = o.stats(d, c)
                st.append([s.open_count, s.flappy_count, s.ctcss_count, s.no_ctcss_count, s.active_counter])
            out[f"counts{d}"] = np.array(st, np.int64)
        path = os.path.join(HERE, name + ".npz")
        np.savez_compressed(path, **out)
        print(name, os.path.getsize(path), "bytes")
    import test_oracle_leaf_vs_ref as leaf
    import test_oracle_scan as scan
    ref = {}
    ref.update(leaf.reference_outputs())
    ref.update(scan.reference_outputs())
    ref = {k: sha256(v) for k, v in ref.items()}
    path = os.path.join(HERE, "ref_leaf.npz")
    np.savez_compressed(path, **ref)
    print("ref_leaf", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
