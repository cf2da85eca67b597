"""Helper of test_gpu_conv3d_down.py (run as a subprocess): builds the UNMODIFIED reference low-res discriminator (staged at
oracle/_ref/src) with this repository's ops and runs logits, the R1 input gradient (double backward) and the parameter
gradients. argv: <out file> <mode>; mode 'base' (F.conv3d on the engine), 'ours' (also conv3d_down.install), 'truth'
(float64 blocks on the CPU), 'profile' ('ours' under torch.profiler: kernel names, and the output shapes of every engine forward
call with its kernel size, next to the full-resolution output shapes of the 1x1x1 downsampling layers, which take the
decomposition)."""
import sys
import types
import warnings

import torch

warnings.filterwarnings('ignore')
sys.modules.setdefault('imageio', types.ModuleType('imageio'))
from model import discriminator_lres      # noqa: E402
from torch_utils import custom_ops        # noqa: E402
from torch_utils.ops import conv_nd, conv3d_down  # noqa: E402

out_file, mode = sys.argv[1], sys.argv[2]
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False
if mode != 'truth':
    conv_nd.install_functional(discriminator_lres)
if mode in ('ours', 'profile'):
    assert conv3d_down.install(discriminator_lres) == [discriminator_lres.Conv3dLayer]

torch.manual_seed(2)
D = discriminator_lres.VideoDiscriminator(seq_length=16, max_edge=64, num_fp16_res=0)
x = torch.rand(2, 3, 16, 64, 64, generator=torch.Generator().manual_seed(12)) * 2 - 1
if mode == 'truth':
    # the blocks in float64; the epilogue casts its input to float32 (discriminator_lres.py:400) and stays fp32 (CPU SIMT)
    D = D.double()
    D.epilogue.float()
    for m in D.modules():                  # upfirdn2d takes float32 filters
        for name, buf in m.named_buffers(recurse=False):
            setattr(m, name, buf.float())
    x = x.double()
else:
    D, x = D.cuda(), x.cuda()
x.requires_grad_(True)


def step():
    logits = D(x)
    gx, = torch.autograd.grad(logits.sum(), [x], create_graph=True)
    (gx.square().sum() + torch.nn.functional.softplus(logits).mean()).backward()
    return logits, gx


if mode == 'profile':
    full, seen = [], []
    for m in D.modules():
        if type(m).__name__ == 'Conv3dLayer' and (m.spatial_down or m.temporal_down) and conv3d_down.faster(m.weight.shape):
            m.register_forward_hook(lambda mod, inp, o: full.append([inp[0].shape[0], mod.out_channels, *inp[0].shape[2:], 1, 1, 1]))
    fprop = custom_ops.ConvNdPlugin.fprop

    def logged(self, x_, w_, *a, **k):
        y = fprop(self, x_, w_, *a, **k)
        seen.append(list(y.shape) + list(w_.shape[2:]))             # output shape and kernel size
        return y
    custom_ops.ConvNdPlugin.fprop = logged
    step()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    names = sorted({e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA})
    torch.save({'kernels': names, 'full': full, 'fprop': seen}, out_file)
    sys.exit(0)

logits, gx = step()
grads = torch.cat([p.grad.flatten().double() for p in D.parameters() if p.grad is not None])
torch.save({'logits': logits.detach().double().cpu(), 'r1_gx': gx.detach().double().cpu(), 'grad': grads.double().cpu()}, out_file)
