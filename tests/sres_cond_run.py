"""Helper of test_sres_cond_host.py / test_gpu_sres_cond.py (run as a subprocess): the UNMODIFIED reference super-res
generator (staged at oracle/_ref/src) with torch_utils.ops.sres_cond.

  plan     the plans evaluated in float64 (sres_cond.evaluate) against the reference's prep_cond for the default G
           (hr 144 x 256, lr 36 x 64), the class default (256 x 256, 32 x 32), temporal_context 2, margin_size 6 and
           fourfeats=True
  install  install() is idempotent, reaches classes persistence rebuilt from a pickle, leaves CPU forwards bitwise
           unchanged, and applies() rejects what it must
  layers   (cuda) the inputs of every layer of the default G at N T = 64 as the reference builds them, and the plans
  model    (cuda) the installed generator against the not-installed one (both with modulated_conv.install): outputs,
           parameter gradients, a second-order gradient through x_prev, magnitude_ema / w_avg after a beta 0.999 pass
  chained  (cuda) lvg_infer.chained.generate_video installed and not installed
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
from torch_utils.ops import sres_cond as sc     # noqa: E402

out_file, mode = sys.argv[1], sys.argv[2]
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False
ORIG = gs.Generator.forward
DEFAULT = dict(hr_height=144, hr_width=256, lr_height=36, lr_width=64)


def lr_video(V, n, t_out, seed=0, device='cpu'):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, 3, t_out + 2 * V.temporal_context, V.lr_height, V.lr_width, generator=g).to(device)


if mode == 'plan':
    res = []
    for kw in (DEFAULT, {}, dict(DEFAULT, temporal_context=2), dict(DEFAULT, margin_size=6), dict(DEFAULT, fourfeats=True),
               dict(lr_height=24, lr_width=40, hr_height=96, hr_width=160)):
        torch.manual_seed(0)
        V = gs.VideoGenerator(**kw)
        G = V.SG3
        lr = lr_video(V, 2, 2, seed=3)
        with torch.no_grad():
            ref = G.prep_cond(lr)
        ps = sc.plans(G, lr.size(3), lr.size(4))
        for i, (r, p) in enumerate(zip(ref, ps)):
            got = sc.evaluate(lr, p)
            res.append(dict(cfg=kw, layer=i, kind=type(G.resamples[i]).__name__, shape_ok=tuple(got.shape) == tuple(r.shape),
                            err=float((got - r.double()).abs().max()) if tuple(got.shape) == tuple(r.shape) else None,
                            scale=float(r.abs().max())))
elif mode == 'install':
    assert sc.install(gs) == [gs.Generator]
    fwd = gs.Generator.forward
    assert fwd is not ORIG and fwd.lvg_sres_cond is ORIG
    assert sc.install(gs) == [gs.Generator] and gs.Generator.forward is fwd
    torch.manual_seed(0)
    V = gs.VideoGenerator(hr_height=48, hr_width=64, lr_height=12, lr_width=16, temporal_context=1)
    assert sc.install(V) == [gs.Generator] and gs.Generator.forward is fwd
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
    assert torch.equal(got, ref)
    assert all(torch.equal(a, b) for a, b in zip(ref_ema, V3.buffers()))
    # a generator that persistence rebuilds from its pickled source has a class of its own
    data = pickle.dumps(V)
    gs.persistence._src_to_module_dict.clear()
    Vp = pickle.loads(data)
    cls2 = type(Vp.SG3)
    assert cls2 is not gs.Generator and cls2.__name__ == 'Generator'
    assert sc.install(torch.nn.ModuleList([Vp])) == [cls2] and cls2.forward.lvg_sres_cond is not None
    orig2 = cls2.forward.lvg_sres_cond
    assert sc.install(Vp) == [cls2] and cls2.forward.lvg_sres_cond is orig2
    # only generators with prep_cond, synthesis and resamples are matched
    class Generator(torch.nn.Module):
        def forward(self, x):
            return x
    assert sc.install(Generator()) == []
    # applies(): each rejected case on its own (the device check comes last, so a CPU tensor reports 'cpu' only when it
    # passes every other check)
    G = V.SG3
    reasons = {}
    reasons['cpu'] = sc.rejection(G, lr)
    reasons['fp64'] = sc.rejection(G, lr.double())
    reasons['fp16'] = sc.rejection(G, lr.half())
    with torch.enable_grad():
        reasons['requires_grad'] = sc.rejection(G, lr.clone().requires_grad_(True))
    with torch.no_grad():
        reasons['requires_grad_no_grad_mode'] = sc.rejection(G, lr.clone().requires_grad_(True))
    G_other = copy.deepcopy(G)
    G_other.resamples[3] = torch.nn.Upsample(scale_factor=2)
    reasons['resampler'] = sc.rejection(G_other, lr)
    G_long = copy.deepcopy(G)
    k = next(i for i, r in enumerate(G_long.resamples) if hasattr(r, 'filter'))
    G_long.resamples[k].filter = torch.ones(80) / 80
    reasons['taps'] = sc.rejection(G_long, lr)
    G_wide = copy.deepcopy(G)
    name = G_wide.synthesis.layer_names[5]
    getattr(G_wide.synthesis, name).in_size = np.array([40000, 8])
    reasons['shape'] = sc.rejection(G_wide, lr)
    reasons['short_video'] = sc.rejection(G, lr[:, :, :2])
    # fallbacks run the original method: the patched forward on a CPU call equals ORIG bit for bit (above) and calls it
    calls = []

    def spy(self, *a, **k):
        calls.append(1)
        return ORIG(self, *a, **k)
    with torch.no_grad():
        out = sc._forward(spy)(V3.SG3, z, lr)
    reasons['fallback_calls'] = len(calls)
    gs.Generator.forward = ORIG
    res = reasons
elif mode == 'layers':
    dev = torch.device('cuda')
    torch.manual_seed(0)
    V = gs.VideoGenerator(**DEFAULT).to(dev)
    G = V.SG3
    lr = lr_video(V, 8, 8, seed=1, device=dev)
    with torch.no_grad():
        conds = [c.cpu() for c in G.prep_cond(lr)]
    res = dict(lr=lr.cpu(), conds=conds, plans=[(p.h, p.w, p.window) for p in sc.plans(G, 36, 64)],
               filters=[None if p.filter is None else p.filter.cpu() for p in sc.plans(G, 36, 64)],
               layers=[(int(getattr(G.synthesis, n).in_channels), bool(getattr(G.synthesis, n).use_fp16)) for n in G.synthesis.layer_names])
elif mode in ('model', 'chained'):
    from torch_utils.ops import modulated_conv
    modulated_conv.install(gs)
    dev = torch.device('cuda')
    if mode == 'model':
        torch.manual_seed(0)
        V0 = gs.VideoGenerator(**DEFAULT).to(dev)
        lr = lr_video(V0, 2, 4, seed=2, device=dev)
        res = {}
        for installed in (False, True):
            gs.Generator.forward = ORIG
            if installed:
                sc.install(gs)
            V = copy.deepcopy(V0)
            # forward without gradient, beta 0.999 (update_D's generated pass): output, magnitude_ema, w_avg
            with torch.no_grad():
                torch.manual_seed(3)
                v0 = V(lr, magnitude_ema_beta=0.999)
            bufs = {k: b.detach().cpu().clone() for k, b in V.named_buffers()}
            # forward + backward (update_G's pattern)
            torch.manual_seed(3)
            v = V(lr)
            tgt = torch.randn(v.shape, generator=torch.Generator().manual_seed(11)).to(dev)
            (v * tgt).mean().backward()
            grads = {k: p.grad.detach().cpu().clone() for k, p in V.named_parameters() if p.grad is not None}
            for p in V.parameters():
                p.grad = None
            # second order through the op's backward: the gradient of |d out / d x_prev|^2 (x_prev: layer 2's output, the
            # x_prev of layer 3) with respect to layer 3's weight
            S = V.SG3.synthesis
            L2, L3 = getattr(S, S.layer_names[2]), getattr(S, S.layer_names[3])
            captured = {}
            lay_cls, lay_fwd, lf = type(L2), type(L2).forward, sc.layer_forward

            def spy_cls(self, x, *a, **k):
                y = lay_fwd(self, x, *a, **k)
                if self is L2:
                    captured['x'] = y
                return y

            def spy_op(L, g, x_prev, *a, **k):
                y = lf(L, g, x_prev, *a, **k)
                if L is L2:
                    captured['x'] = y
                return y
            lay_cls.forward, sc.layer_forward = spy_cls, spy_op
            try:
                torch.manual_seed(3)
                v = V(lr)
            finally:
                lay_cls.forward, sc.layer_forward = lay_fwd, lf
            g1, = torch.autograd.grad((v * tgt).sum(), [captured['x']], create_graph=True)
            g2, = torch.autograd.grad(g1.float().square().sum(), [L3.weight])
            res[installed] = dict(v0=v0.cpu(), v=v.detach().cpu(), bufs=bufs, grads=grads, g2=g2.cpu())
        gs.Generator.forward = ORIG
    else:
        from torch_utils.ops import bias_act
        from lvg_infer.chained import generate_video
        from model import generator_lres
        from torch_utils.ops import conv_nd
        assert bias_act._init()
        conv_nd.install_functional(generator_lres)
        torch.manual_seed(0)
        lres_G = generator_lres.VideoGenerator(out_height=36, out_width=64, num_fp16_layers=0, temporal_padding=8,
                                               temporal_emb_dim=1024).to(dev).eval().requires_grad_(False)
        sres_G = gs.VideoGenerator(**DEFAULT).to(dev).eval().requires_grad_(False)
        res = {}
        for installed in (False, True):
            for graph in (False, True):
                gs.Generator.forward = ORIG
                if installed:
                    sc.install(sres_G)
                gen = torch.Generator('cuda').manual_seed(49)
                lr, chunks = generate_video(lres_G, sres_G, 40, generator=gen, segment_length=8, segments_per_batch=2,
                                            as_uint8=False, graph=graph)
                res[(installed, graph)] = torch.cat([f.clone() for _, f in chunks], dim=1)
        gs.Generator.forward = ORIG
torch.save(res, out_file)
