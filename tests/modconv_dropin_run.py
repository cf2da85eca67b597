"""Helper of test_gpu_modconv.py (run as a subprocess on the GPU box): the UNMODIFIED reference generators (staged at
oracle/_ref/src) forward + backward on cuda, as tests/dropin_cuda_run.py builds them. LVG_REF_PLUGINS=1: the reference's own
ops and CUDA plugins; otherwise this repository's ops, and LVG_MODCONV_INSTALL=1 additionally hands the generators'
modulated convolutions to torch_utils.ops.modulated_conv. Saves outputs, parameter gradients and the super-res G's peak
memory."""
import os
import sys
import types
import warnings

import torch

warnings.filterwarnings('ignore')
sys.modules.setdefault('imageio', types.ModuleType('imageio'))
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

import torch_utils.custom_ops as _co            # noqa: E402
if os.environ.get('LVG_REF_PLUGINS') == '1':
    sys.path.append(ROOT)
    from oracle import ref_cuda
    ref_cuda.patch_custom_ops(_co)
from model import generator_lres, generator_sres   # noqa: E402

out = {'installed': []}
if os.environ.get('LVG_REF_PLUGINS') != '1':
    from torch_utils.ops import conv_nd
    assert conv_nd.install_functional(generator_lres) == [generator_lres]
    if os.environ.get('LVG_MODCONV_INSTALL') == '1':
        from torch_utils.ops import modulated_conv
        out['installed'] = [m.__name__ for m in modulated_conv.install(generator_sres, generator_lres)]
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False
dev = torch.device('cuda')


def grads(net):
    return torch.cat([p.grad.flatten().float() for p in net.parameters() if p.grad is not None])


torch.manual_seed(0)
G = generator_lres.VideoGenerator(out_height=36, out_width=64, num_fp16_layers=0, temporal_padding=8, temporal_emb_dim=1024).to(dev)
torch.manual_seed(1)
v = G(2, 32)
out['lres_G'] = v.detach().cpu()
tgt = torch.randn(v.shape, generator=torch.Generator().manual_seed(11)).to(dev)
(v * tgt).mean().backward()
out['lres_G_grad'] = grads(G).cpu()
del G, v

FP16_RES = 0 if os.environ.get('LVG_FP32') == '1' else 4
torch.manual_seed(3)
S = generator_sres.VideoGenerator(hr_height=144, hr_width=256, lr_height=36, lr_width=64, temporal_context=4, num_fp16_res=FP16_RES,
                                  fourfeats=False).to(dev)
lr = (torch.rand(2, 3, 2 + 8, 36, 64, generator=torch.Generator().manual_seed(13)) * 2 - 1).to(dev)
torch.cuda.synchronize()
torch.cuda.reset_peak_memory_stats()
base = torch.cuda.memory_allocated()
hr = S(lr)
out['sres_G'] = hr.detach().float().cpu()
tgt = torch.randn(hr.shape, generator=torch.Generator().manual_seed(14)).to(dev)
(hr.float() * tgt).sum().backward()
torch.cuda.synchronize()
out['sres_peak_bytes'] = torch.cuda.max_memory_allocated() - base
out['sres_G_grad'] = grads(S).cpu()
torch.save(out, sys.argv[1])
