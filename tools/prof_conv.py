"""Launch each wgmma convolution kernel (fprop with fused BatchNorm statistics / dgrad / wgrad) and the BatchNorm kernels a few
times on ResNet-18 layer shapes -- the ncu target (`tools/gpu_ci.sh ncu_conv`)."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from draco_b200.ops import conv as C  # noqa: E402
from draco_b200.ops import norm as NM  # noqa: E402

dev = torch.device("cuda", 0)


def cl(t):
    return t.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)


for (n, c, k, hw) in [(128, 64, 64, 32), (128, 128, 128, 16), (128, 256, 256, 8)]:
    x = cl(torch.randn(n, c, hw, hw, device=dev))
    w = (torch.randn(k, c, 3, 3, device=dev) * 0.05).to(torch.bfloat16).permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
    dy = cl(torch.randn(n, k, hw, hw, device=dev))
    bn = NM.FusedBatchNorm2d(k).to(dev)
    for _ in range(3):
        req = C.BnStatRequest(1e-5, 0.1)
        if C.halo_supported(hw, hw, c, k):
            y = C.conv3x3_halo(x, w, False, None, req)
            C.conv3x3_halo(dy, w, True)
        else:
            y = C.convg_tcgen05(x, w, (hw, hw), 1, False, None, req)
            C.convg_tcgen05(dy, w, (hw, hw), 1, True)
        C.convg_wgrad_tcgen05(dy, x, 3, 1)
        yg = y.clone().requires_grad_(True)
        z = bn(yg, relu=True)
        z.backward(dy)
    torch.cuda.synchronize()
x = cl(torch.randn(128, 3, 32, 32, device=dev))
w = (torch.randn(64, 3, 3, 3, device=dev) * 0.2).to(torch.bfloat16).permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
dy = cl(torch.randn(128, 64, 32, 32, device=dev))
for _ in range(3):
    C.conv_stem_fprop(x, w, None, C.BnStatRequest(1e-5, 0.1))
    C.conv_stem_wgrad(dy, x)
torch.cuda.synchronize()
print("done")
