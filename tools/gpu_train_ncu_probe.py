"""One launch of every non-GEMM kernel of the training step at Latte-XL/2, local batch 5 (for `ncu --set full`)."""
import sys
import torch
sys.path.insert(0, ".")
from latte_b200.train_ops import NativeOps

dev = torch.device("cuda:0")
ops = NativeOps(torch.bfloat16)
B, rpb, D = 5, 4096, 1152
T = B * rpb
g = torch.Generator().manual_seed(0)
dx = torch.randn(T, D, generator=g).to(dev)
x = torch.randn(T, D, generator=g).to(dev)
m16 = torch.randn(T, D, generator=g).to(dev).bfloat16()
u = torch.randn(T, 4 * D, generator=g).to(dev).bfloat16()
da = torch.randn(T, 4 * D, generator=g).to(dev).bfloat16()
mod = torch.randn(B, 6 * D, generator=g).to(dev)
dmod = torch.zeros(B, 6 * D, device=dev)
db = torch.zeros(4 * D, device=dev)
qkv = torch.randn(T, 3 * D, generator=g).to(dev).bfloat16()
do = torch.randn(T, D, generator=g).to(dev).bfloat16()
for rep in range(2):
    o = ops.attention(qkv, B, 16, 256, 16, False)
    ops.attention_bwd(qkv, o, do, B, 16, 256, 16, False)
    ops.attention_bwd(qkv, o, do, B, 16, 256, 16, True)
    ops.ln_modulate_bwd(m16, x, mod[:, :D], mod[:, D:2 * D], rpb, dx, dmod[:, :D], dmod[:, D:2 * D])
    ops.gate_bwd(dx, m16, mod[:, 2 * D:3 * D], rpb, dmod[:, 2 * D:3 * D], db[:D])
    ops.gelu_bwd(da, u, db)
    ops.colsum(qkv, db[:3 * D])
torch.cuda.synchronize()
print("done")
