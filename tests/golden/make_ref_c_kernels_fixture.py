"""Writes tests/golden/ref_c_kernels.npz: inputs and outputs of the reference's two C kernels
(lance-linalg/src/simd/f16.c: l2_f16_avx2, dist_table.c: sum_4bit_dist_table_32bytes_batch_avx512),
compiled by oracle/Makefile into oracle/_ref/libref_simd.so.  tests/test_oracle_golden.py compares the
oracle against these stored outputs, so the comparison needs neither the reference sources nor an
AVX-512 host.  Regenerate (needs oracle/_ref and an AVX-512BW CPU):
    python tests/golden/make_ref_c_kernels_fixture.py
"""
import ctypes as C
import json
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ref = C.CDLL(os.path.join(os.path.dirname(os.path.dirname(HERE)), "oracle", "_ref", "libref_simd.so"))
ref.l2_f16_avx2.restype = C.c_float
ref.l2_f16_avx2.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32]
ref.sum_4bit_dist_table_32bytes_batch_avx512.restype = None
ref.sum_4bit_dist_table_32bytes_batch_avx512.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]

out = {}
rng = np.random.default_rng(1)
for d in (8, 16, 128, 130, 768):
    x = rng.standard_normal(d).astype(np.float16)
    y = rng.standard_normal(d).astype(np.float16)
    out[f"l2_f16_x_{d}"], out[f"l2_f16_y_{d}"] = x, y
    out[f"l2_f16_out_{d}"] = np.float32(ref.l2_f16_avx2(x.ctypes.data, y.ctypes.data, d))

cases = [(np.asarray(c["codes"], np.uint8), np.asarray(c["dist_table"], np.uint8), c["code_len"])
         for c in json.load(open(os.path.join(HERE, "reference_known_answers.json")))
         if c["op"] == "sum_4bit_dist_table"]
rng = np.random.default_rng(7)
for code_len in (2, 4, 8, 16):  # the C kernel consumes 64 code bytes (= 2 sub-vector pairs) per step
    cases.append((rng.integers(0, 256, 32 * code_len, dtype=np.uint8),
                  rng.integers(0, 256 // (2 * code_len), 32 * code_len, dtype=np.uint8), code_len))
for i, (codes, table, code_len) in enumerate(cases):
    res = np.zeros(32, np.uint16)
    ref.sum_4bit_dist_table_32bytes_batch_avx512(codes.ctypes.data, codes.size, table.ctypes.data, res.ctypes.data)
    out[f"dt_codes_{i}"], out[f"dt_table_{i}"], out[f"dt_out_{i}"] = codes, table, res
    out[f"dt_code_len_{i}"] = np.int64(code_len)
out["dt_cases"] = np.int64(len(cases))
np.savez_compressed(os.path.join(HERE, "ref_c_kernels.npz"), **out)
