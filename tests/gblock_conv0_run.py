"""Helper of test_gblock_conv0_host.py / test_gpu_gblock_conv0.py (run as a subprocess): the UNMODIFIED reference low-res
generator (staged at oracle/_ref/src) with torch_utils.ops.gblock_conv0.

  install  install() is idempotent and chains with gblock_tail, modulated_conv and lres_torgb in every order, reaches
           classes persistence rebuilt from a pickle, runs the replaced method bit for bit outside the envelope, and both
           block forwards (with and without gblock_tail) reproduce the reference bit for bit with the reference head
  G        the whole default G with conv_nd's functional install, without the fused installs, with modulated_conv,
           gblock_tail and lres_torgb, and with those and gblock_conv0: forward + backward at beta 1, the frozen beta 0.999
           forward (update_D's generated pass) and an inference forward; no host synchronisation; the kernels the profiler
           sees for the last block in each mode, and which calls the install routes to the op
"""
import copy
import itertools
import pickle
import sys
import types
import warnings

import torch

warnings.filterwarnings('ignore')
sys.modules.setdefault('imageio', types.ModuleType('imageio'))

from model import generator_lres as gl             # noqa: E402
from torch_utils.ops import _install                # noqa: E402
from torch_utils.ops import gblock_conv0 as gc      # noqa: E402
from torch_utils.ops import gblock_tail as gt       # noqa: E402
from torch_utils.ops import lres_torgb as lt        # noqa: E402
from torch_utils.ops import modulated_conv as mc    # noqa: E402

out_file, mode = sys.argv[1], sys.argv[2]
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False
ORIG_TORGB = gl.ToRGB.forward
ORIG = gl.Synthesis3dResBlock.forward
ORIG_TMC = gl.temporal_modulated_conv3d


def reset():
    gl.ToRGB.forward = ORIG_TORGB
    gl.Synthesis3dResBlock.forward = ORIG
    gl.temporal_modulated_conv3d = ORIG_TMC


def chain(fn):
    names = []
    while fn is not None:
        names.append(next((a for a in ('lvg_gblock_conv0', 'lvg_gblock_tail') if hasattr(fn, a)), 'model'))
        fn = getattr(fn, '__wrapped__', None)
    return names


def install_all():
    reset()
    mc.install(gl)
    gt.install(gl)
    lt.install(gl)
    gc.install(gl)


if mode == 'install':
    res = {}
    installs = {'conv0': lambda: gc.install(gl), 'tail': lambda: gt.install(gl), 'modconv': lambda: mc.install(gl),
                'torgb': lambda: lt.install(gl)}
    for order in itertools.permutations(installs):
        reset()
        for k in order + order:                                   # each twice: idempotent
            installs[k]()
        res[order] = (sorted(chain(gl.Synthesis3dResBlock.forward)), gl.temporal_modulated_conv3d is mc.temporal_modulated_conv3d,
                      _install.find(gl.ToRGB.forward, 'lvg_lres_torgb') is not None)
    reset()
    assert gc.install(gl) == [gl.Synthesis3dResBlock]
    fwd = gl.Synthesis3dResBlock.forward
    torch.manual_seed(0)
    B = gl.Synthesis3dResBlock(16, 8, out_channels=8, temporal_ksize=3, spatial_ksize=3, temporal_up=True, spatial_up=True)
    assert gc.install(B) == [gl.Synthesis3dResBlock] and gl.Synthesis3dResBlock.forward is fwd
    # a block that persistence rebuilds from its pickled source has a class of its own
    data = pickle.dumps(B)
    gl.persistence._src_to_module_dict.clear()
    B2 = pickle.loads(data)
    cls2 = type(B2)
    res['pickled'] = cls2 is not gl.Synthesis3dResBlock and gc.install(torch.nn.ModuleList([B2])) == [cls2] and \
        cls2.forward.lvg_gblock_conv0 is not None and gc.install(B2) == [cls2]
    reset()
    # outside the envelope the replaced method runs, bit for bit: CPU tensors and fp64
    calls = []

    def spy(self, *a, **k):
        calls.append(1)
        return ORIG(self, *a, **k)
    patched = gc._forward(spy)
    x = torch.randn(2, 8, 3, 4, 5)
    lat = torch.randn(2, 16, 3)
    bitwise = []
    for beta in (1.0, 0.9):
        a, b = copy.deepcopy(B), copy.deepcopy(B)
        got = patched(a, x, lat, beta)
        ref = ORIG(b, x, lat, beta)
        bitwise.append(torch.equal(got, ref) and all(torch.equal(p, q) for p, q in zip(a.buffers(), b.buffers())))
    Bd = gl.Synthesis3dResBlock(16, 8, temporal_ksize=3, spatial_ksize=3).double()        # (resampling filters stay fp32)
    got = patched(Bd, x.double(), lat.double(), 1.0, None, torch.float64)
    bitwise.append(torch.equal(got, ORIG(Bd, x.double(), lat.double(), 1.0, None, torch.float64)))
    res['cpu_bitwise'] = all(bitwise)
    res['fallback_calls'] = len(calls)
    res['supported'] = [gc.supported(x, torch.float32, tuple(B.weight_0.shape), B.padding, 'lrelu'),
                        gc.supported(x.double(), torch.float64, tuple(B.weight_0.shape), B.padding, 'lrelu')]
    # the block forwards the install runs, with the reference's head (the CPU stand-in for the op): bit for bit the
    # reference without gblock_tail, and bit for bit gblock_tail's own block forward with it
    g = gl.__dict__
    same = []
    for beta in (1.0, 0.9):
        a, b, c, d = (copy.deepcopy(B) for _ in range(4))
        ref = ORIG(a, x, lat, beta, 6)
        got = gc.block_forward(b, g, x, lat, beta, 6, head=gt.head)
        tail_ref = gt.block_forward(c, g, x, lat, beta, 6)
        tail_got = gt.block_forward(d, g, x, lat, beta, 6, head=gt.head)
        same.append(torch.equal(got, ref) and torch.equal(tail_got, tail_ref)
                    and all(torch.equal(p, q) for p, q in zip(a.buffers(), b.buffers())))
    res['block_forward_bitwise'] = all(same)
    reset()
elif mode == 'G':
    from torch_utils.ops import conv_nd
    conv_nd.install_functional(gl)
    dev = torch.device('cuda')
    torch.manual_seed(0)
    G0 = gl.VideoGenerator(out_height=36, out_width=64).to(dev)

    def step(G, beta, seed=1):
        torch.manual_seed(seed)
        v = G(2, 32, magnitude_ema_beta=beta)
        tgt = torch.randn(v.shape, generator=torch.Generator().manual_seed(11)).to(dev)
        (v * tgt).mean().backward()
        grads = {n: p.grad.float().cpu() for n, p in G.named_parameters() if p.grad is not None}
        for p in G.parameters():
            p.grad = None
        return v.detach().cpu(), grads

    res = {}
    for ours in ('none', 'three', 'four'):
        reset()
        if ours == 'three':
            mc.install(gl)
            gt.install(gl)
            lt.install(gl)
        elif ours == 'four':
            install_all()
        r = {}
        G = copy.deepcopy(G0)
        v, g = step(G, 1.0)
        r['train'] = dict(v=v, g=g, bufs={n: b.cpu() for n, b in G.named_buffers()})
        G = copy.deepcopy(G0).requires_grad_(False)
        torch.manual_seed(1)
        v = G(2, 32, magnitude_ema_beta=0.999)                      # update_D's generated pass
        r['gen'] = dict(v=v.cpu(), bufs={n: b.cpu() for n, b in G.named_buffers()})
        with torch.no_grad():
            torch.manual_seed(1)
            r['infer'] = dict(v=G0(2, 32).cpu())
        res[ours] = r
    # installed: no host synchronisation
    install_all()
    G = copy.deepcopy(G0)
    step(G, 1.0)
    Gf = copy.deepcopy(G0).requires_grad_(False)
    Gf(2, 32, magnitude_ema_beta=0.999)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        torch.manual_seed(1)
        v = G(2, 32)
        v.square().mean().backward()
        Gf(2, 32, magnitude_ema_beta=0.999)
        res['nosync'] = True
    except RuntimeError as e:
        res['nosync'] = str(e)
    torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()

    # the kernels of each mode, for the generator's last block (64 channels) as the installed G calls it
    feats = {}

    def grab(self, input, latent, *a, **k):
        feats['in'] = (input.detach(), latent.detach(), a, k)
        return ORIG(self, input, latent, *a, **k)
    reset()
    gl.Synthesis3dResBlock.forward = grab
    with torch.no_grad():
        G0(2, 32)
    install_all()
    xin, lat, args, kwargs = feats['in']
    B = copy.deepcopy(G0.spatial_layers[-1])

    def profile(fn):
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]

    def train():
        xx = xin.clone().requires_grad_(True)
        B(xx, lat, 1.0, *args[1:], **kwargs).square().sum().backward()

    def gen():
        Bf = copy.deepcopy(B).requires_grad_(False)
        Bf(xin, lat, 0.999, *args[1:], **kwargs)

    def infer():
        with torch.no_grad():
            B(xin, lat, 1.0, *args[1:], **kwargs)
    res['prof'] = {name: profile(fn) for name, fn in (('train', train), ('gen', gen), ('infer', infer))}
    dt = kwargs.get('dtype')
    with torch.no_grad():
        routed_infer = gc._takes(B, xin, lat, 1.0, dt) is not None
    res['routed'] = {'train': gc._takes(B, xin.clone().requires_grad_(True), lat, 1.0, dt) is not None,
                     'gen': gc._takes(copy.deepcopy(B).requires_grad_(False), xin, lat, 0.999, dt) is not None,
                     'infer': routed_infer}
    # every block of the G: the calls the install routes to the op in update_G
    res['routed_train'] = [gc._takes(b, torch.zeros(1, b.in_channels, 1, 4, 4, device=dev), torch.zeros(1, b.latent_dim, 1, device=dev))
                           is not None for b in list(G0.temporal_layers) + list(G0.spatial_layers)]
    reset()
torch.save(res, out_file)
