"""Runs each hot kernel a few times at a model shape so that ncu can capture it:
   ncu --set full --clock-control none --import-source on -k regex:<pattern> -s <skip> -c 1 -o gpurun_out/<name> python tools/profile_kernels.py <what>
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'long-video-gan_b200'))
from torch_utils.ops import bias_act, upfirdn2d, filtered_lrelu  # noqa: E402

DEV = 'cuda'
what = sys.argv[1] if len(sys.argv) > 1 else 'all'
reps = 3


def run(name, fn):
    if what in ('all', name):
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()


x = torch.randn(8, 64, 160, 36, 64, device=DEV)
b = torch.randn(64, device=DEV)
xg, bg = x.clone().requires_grad_(True), b.clone().requires_grad_(True)
run('bias_act_fwd', lambda: bias_act.bias_act(xg, bg, act='lrelu', clamp=256))      # as in a training step: writes the 2-bit codes
run('bias_act_fwd_nograd', lambda: bias_act.bias_act(x, b, act='lrelu', clamp=256))
y = bias_act.bias_act(xg, bg, act='lrelu', clamp=256)
dy = torch.randn_like(y)
run('bias_act_bwd', lambda: torch.autograd.grad(y, [xg, bg], dy, retain_graph=True))
del x, xg, y, dy

f4 = upfirdn2d.setup_filter([1, 3, 3, 1], separable=True).to(DEV)
x = torch.randn(8, 8192, 18, 32, device=DEV)
run('upfirdn_up2', lambda: upfirdn2d.upfirdn2d(x, f4, up=2, padding=[2, 1, 2, 1], gain=4))
x = torch.randn(8, 8192, 64, 64, device=DEV)
run('upfirdn_down2', lambda: upfirdn2d.upfirdn2d(x, f4, down=2, padding=[1, 1, 1, 1]))
lin = (torch.tensor([1., 3., 3., 1.], device=DEV) / 8)[:, None]
x = torch.randn(8, 256, 80, 144, device=DEV)
run('upfirdn_tup', lambda: upfirdn2d.upfirdn2d(x, lin, up=[1, 2], padding=[0, 0, 2, 1], gain=2))
del x

k12 = torch.randn(12, device=DEV) / 3
x = torch.randn(16, 128, 166, 278, device=DEV, dtype=torch.float16)
bb = torch.randn(128, device=DEV, dtype=torch.float16)
run('flrelu_u2d2', lambda: filtered_lrelu.filtered_lrelu(x, k12, k12, bb, up=2, down=2, padding=[9, 8, 9, 8], clamp=256))

from torch_utils import custom_ops  # noqa: E402
from torch_utils.ops import conv2d_gradfix  # noqa: E402
convnd = custom_ops.get_plugin('convnd_plugin')
xc =torch.randn(1, 16 * 539, 92, 148, device=DEV, dtype=torch.float16)
wc = torch.randn(16 * 512, 539, 3, 3, device=DEV, dtype=torch.float16) / 70
run('conv_l8', lambda: conv2d_gradfix.conv2d(xc, wc, padding=2, groups=16))
yc = conv2d_gradfix.conv2d(xc, wc, padding=2, groups=16)
dyc = torch.randn_like(yc)
run('conv_wgrad_l8', lambda: convnd.wgrad(xc, dyc, tuple(wc.shape), (2, 2), 16))
