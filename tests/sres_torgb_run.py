"""Helper of test_sres_torgb_host.py / test_gpu_sres_torgb.py (run as a subprocess): the UNMODIFIED reference super-res
generator (staged at oracle/_ref/src) with torch_utils.ops.sres_torgb.

  install  install() is idempotent, reaches classes persistence rebuilt from a pickle, composes with sres_cond.install,
           sres_layer.install and modulated_conv.install in any order (one wrapper each, and every order hands
           generator_forward the same step and ToRGB forward for a call with a backward, a forward-only call and a
           forward-only call with update_emas), leaves CPU forwards bitwise unchanged, and rejection() names each case
  model    (cuda) modulated_conv + sres_cond installed, with and without sres_torgb: the update_emas forward (beta 0.999,
           recording a graph) with the buffers and the statistic sres_layer.mean_sq gave, forward + backward with
           parameter gradients, and lvg_infer.chained.generate_video with sres_layer installed as well
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

from model import generator_sres as gs          # noqa: E402
from torch_utils.ops import modulated_conv      # noqa: E402
from torch_utils.ops import sres_cond as sc     # noqa: E402
from torch_utils.ops import sres_layer as sl    # noqa: E402
from torch_utils.ops import sres_torgb as st    # noqa: E402

out_file, mode = sys.argv[1], sys.argv[2]
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False
ORIG = gs.Generator.forward
DEFAULT = dict(hr_height=144, hr_width=256, lr_height=36, lr_width=64)
OPS = {'torgb': st, 'layer': sl, 'cond': sc}
ATTRS = ('lvg_sres_torgb', 'lvg_sres_layer', 'lvg_sres_cond')


def lr_video(V, n, t_out, seed=0, device='cpu'):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, 3, t_out + 2 * V.temporal_context, V.lr_height, V.lr_width, generator=g).to(device)


def chain(fn):
    """The attributes naming the wrappers of ``fn``'s chain, top first."""
    out = []
    while fn is not None:
        out.append(next((a for a in ATTRS if a in fn.__dict__), 'model'))
        fn = getattr(fn, '__wrapped__', None)
    return out


if mode == 'install':
    res = {'chains': {}, 'routes': {}}
    torch.manual_seed(0)
    V = gs.VideoGenerator(hr_height=48, hr_width=64, lr_height=12, lr_width=16, temporal_context=1)
    lr = lr_video(V, 1, 2, seed=4)
    z = torch.randn(1, V.latent_z_dim, generator=torch.Generator().manual_seed(5))
    # every order, each install twice; the CPU stand-in takes every call (the size queries and the device check are the
    # GPU's business) and records what generator_forward is handed
    saved = (sc.applies, sl.rejection, st.rejection, sc.generator_forward)
    seen = []

    def spy_generator_forward(G, g, z, cond, *args, **kwargs):
        seen.append((kwargs.get('step'), kwargs.get('torgb')))
        return torch.zeros([])
    for order in list(itertools.permutations(('torgb', 'layer', 'cond'))) + [('layer', 'cond'), ('torgb', 'cond'),
                                                                            ('cond', 'torgb')]:
        gs.Generator.forward = ORIG
        for op in order + order:
            OPS[op].install(gs)
        modulated_conv.install(gs)
        res['chains'][order] = chain(gs.Generator.forward)
        sc.applies = lambda *a, **k: True
        sl.rejection = st.rejection = lambda *a, **k: None
        sc.generator_forward = spy_generator_forward
        try:
            seen.clear()
            V.SG3(z, lr)                                      # records a backward
            with torch.no_grad():
                V.SG3(z, lr)                                  # forward only
                V.SG3(z, lr, update_emas=True)                # forward only, with the magnitude EMA update
            res['routes'][order] = [(getattr(s, '__module__', None), getattr(t, '__module__', None)) for s, t in seen]
        finally:
            sc.applies, sl.rejection, st.rejection, sc.generator_forward = saved
    gs.Generator.forward = ORIG
    assert st.install(V) == [gs.Generator]
    fwd = gs.Generator.forward
    assert fwd.lvg_sres_torgb is ORIG and st.install(gs) == [gs.Generator] and gs.Generator.forward is fwd
    # CPU forwards are bitwise what they were (the original method runs)
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
    res['pickled'] = st.install(torch.nn.ModuleList([Vp])) == [cls2] and cls2.forward.lvg_sres_torgb is not None
    # rejection(): each case on its own (the device check comes last)
    G = V.SG3
    reasons = {'cpu': st.rejection(G, lr), 'fp64': st.rejection(G, lr.double())}
    with torch.enable_grad():
        reasons['requires_grad'] = st.rejection(G, lr.clone().requires_grad_(True))
    G_k3 = copy.deepcopy(G)
    Lt = getattr(G_k3.synthesis, G_k3.synthesis.layer_names[-1])
    Lt.weight = torch.nn.Parameter(torch.zeros(Lt.weight.shape[0], Lt.weight.shape[1], 3, 3))
    Lt.conv_kernel = 3
    reasons['layer'] = st.rejection(G_k3, lr)
    G_wide = copy.deepcopy(G)
    Lw = getattr(G_wide.synthesis, G_wide.synthesis.layer_names[-1])
    c_lr_window = Lw.in_channels - getattr(G_wide.synthesis, G_wide.synthesis.layer_names[-2]).out_channels
    Lw.in_channels = 1100 + c_lr_window                           # more x_prev channels than the op takes
    Lw.weight = torch.nn.Parameter(torch.zeros(Lw.weight.shape[0], Lw.in_channels, 1, 1))
    reasons['torgb_shape'] = (st.rejection(G_wide, lr), sc.rejection(G_wide, lr))
    res['reasons'] = reasons
    # fallbacks run the replaced method
    calls = []

    def spy(self, *a, **k):
        calls.append(1)
        return ORIG(self, *a, **k)
    with torch.no_grad():
        st._forward(spy)(V3.SG3, z, lr)
    res['fallback_calls'] = len(calls)
    gs.Generator.forward = ORIG
elif mode == 'model':
    modulated_conv.install(gs)
    dev = torch.device('cuda')
    torch.manual_seed(0)
    V0 = gs.VideoGenerator(**DEFAULT).to(dev)
    lr = lr_video(V0, 2, 4, seed=2, device=dev)
    res = {'output_scale': float(V0.SG3.synthesis.output_scale)}
    mean_sq = sl.mean_sq
    for torgb in (False, True):
        gs.Generator.forward = ORIG
        sc.install(gs)
        if torgb:
            st.install(gs)
        V = copy.deepcopy(V0)
        stats = []

        def recording_mean_sq(*a, **k):
            stats.append(mean_sq(*a, **k).clone())
            return stats[-1]
        sl.mean_sq = recording_mean_sq
        try:
            Lt = getattr(V.SG3.synthesis, V.SG3.synthesis.layer_names[-1])
            ema_before = Lt.magnitude_ema.detach().clone()
            # with a recorded graph, so that the installed ToRGB forward takes the op and its update_emas path
            torch.manual_seed(3)
            v0 = V(lr, magnitude_ema_beta=0.999).detach()
        finally:
            sl.mean_sq = mean_sq
        bufs = {k: b.detach().cpu().clone() for k, b in V.named_buffers()}
        torgb_ema = None
        if torgb:
            assert len(stats) == 1
            torgb_ema = stats[0].lerp(ema_before, Lt.magnitude_ema_beta).cpu()
        torch.manual_seed(3)
        v = V(lr)
        tgt = torch.randn(v.shape, generator=torch.Generator().manual_seed(11)).to(dev)
        (v * tgt).mean().backward()
        grads = {k: p.grad.detach().cpu().clone() for k, p in V.named_parameters() if p.grad is not None}
        # chained inference (forward only, eval), sres_layer installed on both sides
        sl.install(gs)
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
        res[torgb] = dict(v0=v0.cpu(), v=v.detach().cpu(), bufs=bufs, grads=grads, chained=chained, torgb_ema=torgb_ema,
                          torgb_name=V.SG3.synthesis.layer_names[-1])
    gs.Generator.forward = ORIG
torch.save(res, out_file)
