"""Driver for ncu captures of the wgmma 3xTF32 dense layer (csrc/mlp_tc.cu).
    ncu --set full --clock-control none --import-source on -k regex:linear_tf32x3 -s 2 -c 1 \
        -o gpurun_out/prof_linear python tools/profile_linear.py
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from librecommender_b200 import _lib  # noqa: E402

R, din, dout = int(os.environ.get("PROF_ROWS", 1 << 19)), 1792, 128
x = torch.randn(R, din, device="cuda")
Wt = torch.randn(dout, din, device="cuda") / din ** 0.5
b = torch.randn(dout, device="cuda")
y = torch.empty(R, dout, device="cuda")
ld = int(_lib.lib.b200_linear_tf32x3_split_ld(din))
ws = torch.empty(2 * dout * ld, device="cuda")
_lib.check(_lib.lib.b200_linear_tf32x3_split_weights(_lib.ptr(Wt), din, din, dout, _lib.ptr(ws), _lib.current_stream()))
for _ in range(4):
    _lib.check(_lib.lib.b200_linear_tf32x3(_lib.ptr(x), din, R, _lib.ptr(Wt), din, _lib.ptr(ws), _lib.ptr(b), din, dout, 1,
                                           _lib.ptr(y), dout, _lib.current_stream()))
torch.cuda.synchronize()
print("done")
