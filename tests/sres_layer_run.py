"""Helper of test_sres_layer_host.py / test_gpu_sres_layer.py (run as a subprocess): the UNMODIFIED reference super-res
generator (staged at oracle/_ref/src) with torch_utils.ops.sres_layer.

  install  install() is idempotent, reaches classes persistence rebuilt from a pickle, composes with sres_cond.install and
           modulated_conv.install in either order, leaves CPU forwards bitwise unchanged, and rejection() names each case
           it must
  model    (cuda) modulated_conv + sres_cond + sres_layer installed against modulated_conv + sres_cond: the update_emas
           forward without gradient (beta 0.999) with the buffers after it, forward + backward with parameter gradients,
           and lvg_infer.chained.generate_video
"""
import copy
import pickle
import sys
import types
import warnings

import numpy as np
import torch

warnings.filterwarnings('ignore')
sys.modules.setdefault('imageio', types.ModuleType('imageio'))

from model import generator_sres as gs          # noqa: E402
from torch_utils.ops import modulated_conv      # noqa: E402
from torch_utils.ops import sres_cond as sc     # noqa: E402
from torch_utils.ops import sres_layer as sl    # noqa: E402

out_file, mode = sys.argv[1], sys.argv[2]
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False
ORIG = gs.Generator.forward
DEFAULT = dict(hr_height=144, hr_width=256, lr_height=36, lr_width=64)


def lr_video(V, n, t_out, seed=0, device='cpu'):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, 3, t_out + 2 * V.temporal_context, V.lr_height, V.lr_width, generator=g).to(device)


def chain(fn):
    """The attributes naming the wrappers of ``fn``'s chain, top first."""
    out = []
    while fn is not None:
        out.append(next((a for a in ('lvg_sres_layer', 'lvg_sres_cond') if a in fn.__dict__), 'model'))
        fn = getattr(fn, '__wrapped__', None)
    return out


if mode == 'install':
    res = {}
    # idempotent, either order with sres_cond; modulated_conv.install patches module globals and composes with both
    for order in (('layer', 'cond'), ('cond', 'layer')):
        gs.Generator.forward = ORIG
        for op in order + order:
            (sl if op == 'layer' else sc).install(gs)
        modulated_conv.install(gs)
        res[order] = chain(gs.Generator.forward)
        # the sres_cond wrapper hands a call the fused op takes to it, wherever it sits
        top = gs.Generator.forward
        assert (sc._install.find(top, 'lvg_sres_layer') is not None) and (sc._install.find(top, 'lvg_sres_cond') is not None)
    gs.Generator.forward = ORIG
    torch.manual_seed(0)
    V = gs.VideoGenerator(hr_height=48, hr_width=64, lr_height=12, lr_width=16, temporal_context=1)
    assert sl.install(V) == [gs.Generator]
    fwd = gs.Generator.forward
    assert fwd.lvg_sres_layer is ORIG and sl.install(gs) == [gs.Generator] and gs.Generator.forward is fwd
    # CPU forwards are bitwise what they were (the original method runs)
    lr = lr_video(V, 1, 2, seed=4)
    z = torch.randn(1, V.latent_z_dim, generator=torch.Generator().manual_seed(5))
    gs.Generator.forward = ORIG
    with torch.no_grad():
        ref = V.SG3(z, lr, update_emas=True)
        ref_ema = [b.clone() for b in V.buffers()]
    gs.Generator.forward = fwd
    torch.manual_seed(0)
    V3 = gs.VideoGenerator(hr_height=48, hr_width=64, lr_height=12, lr_width=16, temporal_context=1)
    with torch.no_grad():
        got = V3.SG3(z, lr, update_emas=True)
    res['cpu_bitwise'] = torch.equal(got, ref) and all(torch.equal(a, b) for a, b in zip(ref_ema, V3.buffers()))
    # a generator that persistence rebuilds from its pickled source has a class of its own
    data = pickle.dumps(V)
    gs.persistence._src_to_module_dict.clear()
    Vp = pickle.loads(data)
    cls2 = type(Vp.SG3)
    assert cls2 is not gs.Generator and cls2.__name__ == 'Generator'
    assert sl.install(torch.nn.ModuleList([Vp])) == [cls2]
    res['pickled'] = cls2.forward.lvg_sres_layer is not None and sl.install(Vp) == [cls2]
    # rejection(): each case on its own (the device check comes last)
    G = V.SG3
    reasons = {}
    reasons['cpu'] = sl.rejection(G, lr)
    reasons['fp64'] = sl.rejection(G, lr.double())
    with torch.enable_grad():
        reasons['requires_grad'] = sl.rejection(G, lr.clone().requires_grad_(True))
    G_other = copy.deepcopy(G)
    G_other.resamples[3] = torch.nn.Upsample(scale_factor=2)
    reasons['resampler'] = sl.rejection(G_other, lr)
    G_wide = copy.deepcopy(G)
    name = G_wide.synthesis.layer_names[5]
    getattr(G_wide.synthesis, name).in_size = np.array([40000, 8])
    reasons['shape'] = sl.rejection(G_wide, lr)
    # a layer only the fused op rejects: a 5 x 5 kernel (more than nine taps per frame) is outside the engine
    G_k5 = copy.deepcopy(G)
    L5 = getattr(G_k5.synthesis, G_k5.synthesis.layer_names[2])
    L5.weight = torch.nn.Parameter(torch.zeros(L5.weight.shape[0], L5.weight.shape[1], 5, 5))
    L5.conv_kernel = 5
    reasons['fused_shape'] = (sl.rejection(G_k5, lr), sc.rejection(G_k5, lr))
    res['reasons'] = reasons
    # fallbacks run the replaced method
    calls = []

    def spy(self, *a, **k):
        calls.append(1)
        return ORIG(self, *a, **k)
    with torch.no_grad():
        sl._forward(spy)(V3.SG3, z, lr)
    res['fallback_calls'] = len(calls)
    gs.Generator.forward = ORIG
elif mode == 'model':
    modulated_conv.install(gs)
    dev = torch.device('cuda')
    torch.manual_seed(0)
    V0 = gs.VideoGenerator(**DEFAULT).to(dev)
    lr = lr_video(V0, 2, 4, seed=2, device=dev)
    res = {}
    for fused in (False, True):
        gs.Generator.forward = ORIG
        sc.install(gs)
        if fused:
            sl.install(gs)
        V = copy.deepcopy(V0)
        with torch.no_grad():
            torch.manual_seed(3)
            v0 = V(lr, magnitude_ema_beta=0.999)
        bufs = {k: b.detach().cpu().clone() for k, b in V.named_buffers()}
        torch.manual_seed(3)
        v = V(lr)
        tgt = torch.randn(v.shape, generator=torch.Generator().manual_seed(11)).to(dev)
        (v * tgt).mean().backward()
        grads = {k: p.grad.detach().cpu().clone() for k, p in V.named_parameters() if p.grad is not None}
        # chained inference (forward only, eval)
        from lvg_infer.chained import generate_video
        from model import generator_lres
        from torch_utils.ops import bias_act, conv_nd
        assert bias_act._init()
        conv_nd.install_functional(generator_lres)
        torch.manual_seed(0)
        lres_G = generator_lres.VideoGenerator(out_height=36, out_width=64, num_fp16_layers=0, temporal_padding=8,
                                               temporal_emb_dim=1024).to(dev).eval().requires_grad_(False)
        sres_G = copy.deepcopy(V0).eval().requires_grad_(False)
        gen = torch.Generator('cuda').manual_seed(49)
        _, chunks = generate_video(lres_G, sres_G, 24, generator=gen, segment_length=8, segments_per_batch=2, as_uint8=False)
        chained = torch.cat([f.clone() for _, f in chunks], dim=1).cpu()
        res[fused] = dict(v0=v0.cpu(), v=v.detach().cpu(), bufs=bufs, grads=grads, chained=chained)
    gs.Generator.forward = ORIG
torch.save(res, out_file)
