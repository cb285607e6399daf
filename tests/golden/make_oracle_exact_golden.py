"""Writes tests/golden/oracle_exact.npz: inputs and every output of the plain-C oracle's exact forward and backward
(bigru_ref_forward / bigru_ref_backward) at two tiny shapes, one with an initial state.  The fixture pins those functions
bit for bit, so a change to the oracle (such as its rounding modes) cannot move the exact restatement unnoticed.

    python tests/golden/make_oracle_exact_golden.py [path/to/libbigru_oracle.so]

The committed file was written by the oracle as it was before the rounding modes were added."""
import ctypes as C
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import oracle_c  # noqa: E402

SHAPES = {"a": (3, 5, 7, 6, 2, 3, 2, True), "b": (4, 6, 9, 8, 3, 2, 1, False)}   # B, T, F, H, L, C, D, h0


def main(so):
    lib = C.CDLL(so)
    lib.bigru_ref_param_count.restype = C.c_int64
    lib.bigru_ref_stash_doubles.restype = C.c_int64
    p = oracle_c._p
    out = {}
    for name, (B, T, F, H, L, C_, D, use_h0) in SHAPES.items():
        rng = np.random.default_rng(sum(map(ord, name)))
        flat = (rng.standard_normal(lib.bigru_ref_param_count(F, H, L, C_, D)) * 0.4).astype(np.float32)
        x = rng.standard_normal((B, T, F)).astype(np.float32)
        h0 = (rng.standard_normal((L * D, B, H)) * 0.5).astype(np.float32) if use_h0 else None
        dl = rng.standard_normal((B, C_)).astype(np.float32)
        logits, hn = np.zeros((B, C_), np.float32), np.zeros((L * D, B, H), np.float32)
        stash = np.zeros(lib.bigru_ref_stash_doubles(B, T, F, H, L, C_, D), np.float64)
        assert lib.bigru_ref_forward(B, T, F, H, L, C_, D, p(flat), p(x), p(h0), p(logits), p(hn), p(stash, C.c_double)) == 0
        grads, dx, dh0 = np.zeros_like(flat), np.zeros_like(x), np.zeros((L * D, B, H), np.float32)
        assert lib.bigru_ref_backward(B, T, F, H, L, C_, D, p(flat), p(x), p(stash, C.c_double), p(dl), p(grads), p(dx), p(dh0)) == 0
        arrs = dict(meta=np.array([B, T, F, H, L, C_, D]), flat=flat, x=x, dlogits=dl, logits=logits, hn=hn, stash=stash,
                    grads=grads, dx=dx, dh0=dh0)
        if h0 is not None:
            arrs["h0"] = h0
        out.update({f"{name}:{k}": v for k, v in arrs.items()})
    np.savez_compressed(os.path.join(HERE, "oracle_exact.npz"), **out)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else oracle_c.build())
