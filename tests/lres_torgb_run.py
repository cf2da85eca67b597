"""Helper of test_lres_torgb_host.py / test_gpu_lres_torgb.py (run as a subprocess): the UNMODIFIED reference low-res
generator (staged at oracle/_ref/src) with torch_utils.ops.lres_torgb.

  install  install() is idempotent, chains with modulated_conv and gblock_tail in every order, reaches classes
           persistence rebuilt from a pickle, and runs the replaced method bit for bit outside the envelope
  layer    the default G's ToRGB layer on cuda: the op's path against the reference forward in the three modes (EMA
           buffer included), the beta != 1 statistic through a fake all_reduce of world size 2, and the gradients of
           the layer's parameters, input and latent against the reference's
  G        the whole default G with modulated_conv + gblock_tail installed, with and without lres_torgb: forward +
           backward at beta 1 and 0.999, no-grad forwards at 0.999, sample_video_segments; no host synchronisation; the
           kernels the profiler sees
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
from torch_utils.ops import gblock_tail as gt       # noqa: E402
from torch_utils.ops import lres_torgb as lt        # noqa: E402
from torch_utils.ops import modulated_conv as mc    # noqa: E402

out_file, mode = sys.argv[1], sys.argv[2]
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False
ORIG = gl.ToRGB.forward
ORIG_BLOCK = gl.Synthesis3dResBlock.forward
ORIG_TMC = gl.temporal_modulated_conv3d


def reset():
    gl.ToRGB.forward = ORIG
    gl.Synthesis3dResBlock.forward = ORIG_BLOCK
    gl.temporal_modulated_conv3d = ORIG_TMC


def chain(fn):
    names = []
    while fn is not None:
        names.append(next((a for a in ('lvg_lres_torgb',) if hasattr(fn, a)), 'model'))
        fn = getattr(fn, '__wrapped__', None)
    return names


if mode == 'install':
    res = {}
    installs = {'torgb': lambda: lt.install(gl), 'modconv': lambda: mc.install(gl), 'tail': lambda: gt.install(gl)}
    for order in itertools.permutations(installs):
        reset()
        for k in order + order:                                   # each twice: idempotent
            installs[k]()
        res[order] = (chain(gl.ToRGB.forward), gl.temporal_modulated_conv3d is mc.temporal_modulated_conv3d,
                      _install.find(gl.Synthesis3dResBlock.forward, 'lvg_gblock_tail') is not None)
    reset()
    assert lt.install(gl) == [gl.ToRGB]
    fwd = gl.ToRGB.forward
    torch.manual_seed(0)
    L = gl.ToRGB(16, 8)
    assert lt.install(L) == [gl.ToRGB] and gl.ToRGB.forward is fwd
    # a layer that persistence rebuilds from its pickled source has a class of its own
    data = pickle.dumps(L)
    gl.persistence._src_to_module_dict.clear()
    L2 = pickle.loads(data)
    cls2 = type(L2)
    res['pickled'] = cls2 is not gl.ToRGB and lt.install(torch.nn.ModuleList([L2])) == [cls2] and \
        cls2.forward.lvg_lres_torgb is not None and lt.install(L2) == [cls2]
    # outside the envelope the replaced method runs, bit for bit: CPU tensors, fp64, LVG_NATIVE_CONV=0
    calls = []

    def spy(self, *a, **k):
        calls.append(1)
        return ORIG(self, *a, **k)
    patched = lt._forward(spy)
    x = torch.randn(2, 8, 3, 4, 5)
    lat = torch.randn(2, 16, 3)
    bitwise = []
    for beta in (1.0, 0.9):
        a, b = copy.deepcopy(L), copy.deepcopy(L)
        got = patched(a, x, lat, beta)
        ref = ORIG(b, x, lat, beta)
        bitwise.append(torch.equal(got, ref) and torch.equal(a.input_magnitude_ema.magnitude_ema, b.input_magnitude_ema.magnitude_ema))
    Ld = copy.deepcopy(L).double()
    got = patched(Ld, x.double(), lat.double(), 1.0, torch.float64)
    bitwise.append(torch.equal(got, ORIG(Ld, x.double(), lat.double(), 1.0, torch.float64)))
    res['cpu_bitwise'] = all(bitwise)
    res['fallback_calls'] = len(calls)
    res['supported'] = [lt.supported(x, torch.float32, tuple(L.weight.shape)), lt.supported(x.double(), torch.float64, (3, 8, 1, 1, 1))]
    reset()
elif mode == 'layer':
    dev = torch.device('cuda')
    torch.manual_seed(0)
    G = gl.VideoGenerator(out_height=36, out_width=64).to(dev)
    L0 = G.to_rgb
    with torch.no_grad():
        L0.bias.copy_(torch.tensor([0.3, -0.2, 0.1]))
        L0.input_magnitude_ema.magnitude_ema.fill_(2.5)
    gen = torch.Generator(device=dev).manual_seed(3)
    x = torch.randn(2, 64, 16, 36, 64, generator=gen, device=dev) * 1.5
    lat = torch.randn(2, 1024, 16, generator=gen, device=dev)
    res = {}
    # forward-only modes: beta 1 and 0.999, fp32 and fp16 layers, against the reference forward
    for dt in (torch.float32, torch.float16):
        for beta in (1.0, 0.999):
            a, b = copy.deepcopy(L0), copy.deepcopy(L0)
            with torch.no_grad():
                ref = ORIG(a, x, lat, beta, dt)
                ours = lt.layer_forward(b, gl.__dict__, x, lat, beta, dt)
            res[('fwd', dt, beta)] = dict(ref=ref.float().cpu(), ours=ours.float().cpu(), dtype=ours.dtype,
                                          ema_ref=float(a.input_magnitude_ema.magnitude_ema), ema_ours=float(b.input_magnitude_ema.magnitude_ema))

    # the statistic goes through all_reduce when dist_sync and the world has two ranks
    class FakeDist:
        class ReduceOp:
            SUM = 'sum'
        calls = []

        @staticmethod
        def all_reduce(t, op):
            FakeDist.calls.append(op)
            t.mul_(2)                                                  # the other rank saw the same statistic
    fake_g = dict(gl.__dict__, dist=FakeDist, dist_utils=types.SimpleNamespace(get_world_size=lambda: 2))
    b = copy.deepcopy(L0)
    with torch.no_grad():
        lt.layer_forward(b, fake_g, x, lat, 0.999, torch.float32)
    res['dist'] = dict(calls=list(FakeDist.calls), ema=float(b.input_magnitude_ema.magnitude_ema),
                       ema_ref=res[('fwd', torch.float32, 0.999)]['ema_ref'])
    # gradients against the reference (fp32 layer): input, latent (through the affine layer), weight, bias
    dy = torch.randn(2, 3, 16, 36, 64, generator=gen, device=dev)
    grads = {}
    for name, fn in (('ref', lambda L, xx, ll: ORIG(L, xx, ll, 1.0, torch.float32)),
                     ('ours', lambda L, xx, ll: lt.layer_forward(L, gl.__dict__, xx, ll, 1.0, torch.float32))):
        runs = []
        for _ in range(2):
            L = copy.deepcopy(L0)
            xx, ll = x.clone().requires_grad_(True), lat.clone().requires_grad_(True)
            y = fn(L, xx, ll)
            y.backward(dy)
            runs.append(dict(x=xx.grad.cpu(), lat=ll.grad.cpu(), w=L.weight.grad.cpu(), b=L.bias.grad.cpu(),
                             aff=L.affine.weight.grad.cpu()))
        grads[name] = runs
    res['grads'] = grads
    # second order: create_graph through the op against the reference
    second = {}
    for name, fn in (('ref', ORIG), ('ours', lambda L, xx, ll, beta, dt: lt.layer_forward(L, gl.__dict__, xx, ll, beta, dt))):
        L = copy.deepcopy(L0)
        xx = x[:, :, :4].clone().requires_grad_(True)
        y = fn(L, xx, lat[:, :, :4], 1.0, torch.float32)
        gx, = torch.autograd.grad((y * dy[:, :, :4]).sum(), [xx], create_graph=True)
        gw, = torch.autograd.grad(gx.square().sum(), [L.weight])
        second[name] = gw.cpu()
    res['second'] = second
    # CUDA-graph capture of forward + backward
    L = copy.deepcopy(L0)
    xs = x.clone().requires_grad_(True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            y = lt.layer_forward(L, gl.__dict__, xs, lat, 1.0, torch.float32)
            y.backward(dy)
    torch.cuda.current_stream().wait_stream(s)
    L.weight.grad = None
    xs.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        yg = lt.layer_forward(L, gl.__dict__, xs, lat, 1.0, torch.float32)
        yg.backward(dy)
    graph.replay()
    torch.cuda.synchronize()
    res['graph'] = dict(y=yg.detach().cpu(), x=xs.grad.cpu(), y_ref=res[('fwd', torch.float32, 1.0)]['ours'],
                        x_ref=grads['ours'][0]['x'])
elif mode == 'G':
    from torch_utils.ops import conv_nd
    conv_nd.install_functional(gl)
    dev = torch.device('cuda')
    torch.manual_seed(0)
    G0 = gl.VideoGenerator(out_height=36, out_width=64).to(dev)

    def install(ours):
        reset()
        mc.install(gl)
        gt.install(gl)
        if ours:
            lt.install(gl)

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
    for ours in (False, True):
        install(ours)
        r = {}
        for beta in (1.0, 0.999):
            G = copy.deepcopy(G0)
            v, g = step(G, beta)
            r[('train', beta)] = dict(v=v, g=g, bufs={n: b.cpu() for n, b in G.named_buffers()})
        G = copy.deepcopy(G0).requires_grad_(False)
        torch.manual_seed(1)
        v = G(2, 32, magnitude_ema_beta=0.999)                      # update_D's generated pass
        r[('gen', 0.999)] = dict(v=v.cpu(), bufs={n: b.cpu() for n, b in G.named_buffers()})
        with torch.no_grad():
            torch.manual_seed(2)
            segs = [s.cpu() for s in G.sample_video_segments(2, 32, segment_length=8)]
        r['segments'] = segs
        res[ours] = r
    # installed: no host synchronisation, and the kernels the profiler sees
    install(True)
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

    def profile(fn):
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]

    # the ToRGB layer alone, as the installed G calls it, in each of the three modes
    feats = {}

    def grab(self, input, latent, *a, **k):
        feats['in'] = (input.detach(), latent.detach())
        return ORIG(self, input, latent, *a, **k)
    reset()
    gl.ToRGB.forward = grab
    with torch.no_grad():
        G0(2, 32)
    install(True)
    xin, lat = feats['in']
    L = copy.deepcopy(G0.to_rgb)

    def train():
        xx = xin.clone().requires_grad_(True)
        L(xx, lat).square().sum().backward()

    def gen():
        Lf = copy.deepcopy(L).requires_grad_(False)
        Lf(xin, lat, 0.999)

    def infer():
        with torch.no_grad():
            L(xin, lat)
    res['prof'] = {name: profile(fn) for name, fn in (('train', train), ('gen', gen), ('infer', infer))}
    reset()
torch.save(res, out_file)
