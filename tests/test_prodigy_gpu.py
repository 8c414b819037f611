"""GPU: the Prodigy step kernels (csrc/prodigy.cu).  Over 150 mixed tensors in one call (bf16 / fp32, 0-D to 4-D,
sizes 1 to 2^20 + 3, views 1-7 elements into guarded buffers, some sets at different offsets mod 16 B): the per-tensor
sums against fp64, m, v, s and p bit-identical to oracle/prodigy_ref.py fed with the kernels' own sums, d, d_max and
d_hat bit-identical to its scalar fold, guard bands untouched, two runs equal bit for bit, a step with every gradient
zero; the emulation bit-identical to the torch-op text on CUDA; no host synchronisation in a whole Prodigy.step() and
no gradient kept past it.  Then a small Flux model (full fine-tune) and a small
Qwen-Image LoRA model train 4 steps with `type = 'Prodigy'` through the engine against the torch-op text stepped in a
second engine, and resume from a checkpoint with the same bits."""
import os
import sys

import pytest
import torch

from oracle import prodigy_ref as P

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
GUARD = 16
SHAPES = [(1,), (7,), (4097,), ((1 << 20) + 3,), (), (17, 241), (32, 3072), (3, 5, 7, 9), (8193,), (2, 8192)]
HYPER = dict(P.DEFAULTS, lr=1.0)
NAMES = ('p', 'g', 'p0', 's', 'm', 'v')


def _bits(t):
    return t.view(torch.int16) if t.dtype == BF16 else t.view(torch.int32) if t.dtype == torch.float32 else t


class Case:
    """one parameter with its state as guarded CUDA views; every fifth case puts p0 one element off the others'
    offset mod 16 B (element-wise path)"""

    def __init__(self, i, shape, dtype, gen):
        self.shape, self.dtype = shape, dtype
        vals = {'p': torch.randn(shape, generator=gen) * 0.05, 'g': torch.randn(shape, generator=gen) * 1e-2,
                'p0': torch.randn(shape, generator=gen) * 0.05, 's': torch.randn(shape, generator=gen) * 1e-8,
                'm': torch.randn(shape, generator=gen) * 1e-9, 'v': torch.rand(shape, generator=gen) * 1e-16}
        off = 1 + i % 7
        self.bufs = {}
        for k, x in vals.items():
            o = off + (1 if k == 'p0' and i % 5 == 0 else 0)
            n = x.numel()
            buf = (torch.randn(o + n + GUARD, generator=gen) * 7).to(dtype).cuda()
            view = buf[o:o + n].view(shape)
            view.copy_(x.to(dtype))
            self.bufs[k] = (buf, view)
        self.views = {k: v for k, (_, v) in self.bufs.items()}
        self.before = {k: v.cpu().clone() for k, v in self.views.items()}
        self.guards0 = {k: b.cpu() for k, (b, _) in self.bufs.items()}

    def guards_intact(self):
        for k, (buf, view) in self.bufs.items():
            off = (view.data_ptr() - buf.data_ptr()) // buf.element_size()
            host, g0 = buf.cpu(), self.guards0[k]
            if not (torch.equal(_bits(host[:off]), _bits(g0[:off]))
                    and torch.equal(_bits(host[off + view.numel():]), _bits(g0[off + view.numel():]))):
                return False
        return True


def _cases(seed=3, count=150):
    gen = torch.Generator().manual_seed(seed)
    small = [s for s in SHAPES if torch.Size(s).numel() < (1 << 20)]
    out = []
    for i in range(count):
        shape = SHAPES[i % len(SHAPES)]
        if i >= 2 * len(SHAPES) and torch.Size(shape).numel() >= (1 << 20):
            shape = small[i % len(small)]
        out.append(Case(i, shape, (BF16, torch.float32)[(i // len(SHAPES)) % 2], gen))
    return out


GS0 = dict(step=4, d=3e-6, d_max=3e-6, d_hat=2e-6, d_numerator=1.5e-9, d_denom=0.0)


def _block(gs):
    from diffusion_pipe_b200 import _abi
    b = torch.zeros(_abi.PRODIGY_STATE_DOUBLES, dtype=torch.float64)
    for k, v in gs.items():
        b[_abi.PRODIGY_SLOTS[k]] = v
    return b.cuda()


def _run(cases, gs=GS0, hyper=HYPER):
    from diffusion_pipe_b200 import ops
    v = [c.views for c in cases]
    args = ops.prodigy_pack([x['p'] for x in v], [x['s'] for x in v], [x['p0'] for x in v], [x['m'] for x in v],
                            [x['v'] for x in v], [0.01 if i % 2 else 0.0 for i in range(len(cases))],
                            [1e-8] * len(cases), [i % 3 == 0 for i in range(len(cases))])
    blk = _block(gs)
    h = {k: hyper[k] for k in ('lr', 'betas', 'beta3', 'd0', 'd_coef', 'growth_rate', 'bias_correction',
                                'safeguard_warmup')}
    ops.prodigy_stats(args, [x['g'] for x in v], blk, **h)
    torch.cuda.synchronize()
    mid = dict(sums=args.scratch[:2 * len(cases)].cpu().view(-1, 2), blk=blk.cpu().clone(),
               m=[c.views['m'].cpu().clone() for c in cases], v=[c.views['v'].cpu().clone() for c in cases],
               s=[c.views['s'].cpu().clone() for c in cases])
    ops.prodigy_apply(args, blk)
    torch.cuda.synchronize()
    return mid, blk.cpu()


@pytest.mark.parametrize('bias_correction', [False, True])
def test_kernels_match_the_specification(bias_correction):
    from diffusion_pipe_b200 import _abi
    S = _abi.PRODIGY_SLOTS
    cases = _cases()
    hyper = dict(HYPER, bias_correction=bias_correction)
    mid, blk = _run(cases, hyper=hyper)
    sc = P.step_scalars(GS0, hyper)
    sums = []
    for i, c in enumerate(cases):
        b = c.before
        m, v, s, dot, a = P.prodigy_stats_emulated(b['p'], b['g'], b['p0'], b['s'], b['m'], b['v'], sc)
        kd, ka = float(mid['sums'][i, 0]), float(mid['sums'][i, 1])
        scale = float((b['g'].double() * (b['p0'].double() - b['p'].double())).abs().sum()) + 1e-300
        assert abs(kd - dot) <= 1e-12 * scale and abs(ka - a) <= 1e-12 * max(a, 1e-300), (i, c.shape, kd, dot)
        for k, want in (('m', m), ('v', v), ('s', s)):
            assert torch.equal(_bits(mid[k][i]), _bits(want)), (i, k, c.shape, c.dtype)
        sums.append((kd, ka))
    new, skipped = P.prodigy_fold(GS0, hyper, sc, sums)
    assert not skipped
    for k in ('d', 'd_max', 'd_hat', 'd_numerator', 'd_denom', 'step'):
        assert float(blk[S[k]]) == new[k], k
    assert float(blk[S['d_lr']]) == sc['d_lr'] and float(blk[S['skip']]) == 0.0
    for i, c in enumerate(cases):
        want = P.prodigy_apply_emulated(c.before['p'], mid['m'][i], mid['v'][i], d_lr=sc['d_lr'], d=new['d'],
                                        eps=1e-8, weight_decay=0.01 if i % 2 else 0.0, fixed_decay=i % 3 == 0)
        assert torch.equal(_bits(c.views['p'].cpu()), _bits(want)), (i, c.shape, c.dtype)
        assert c.guards_intact(), i


def test_two_runs_give_equal_bits():
    outs = []
    for _ in range(2):
        cases = _cases(seed=8, count=70)
        mid, blk = _run(cases)
        outs.append([mid['sums'], blk] + [c.views[k].cpu() for c in cases for k in ('p', 'm', 'v', 's')])
    assert all(torch.equal(_bits(a), _bits(b)) for a, b in zip(*outs))


def test_zero_sums_skip_the_apply_phase():
    from diffusion_pipe_b200 import _abi
    S = _abi.PRODIGY_SLOTS
    cases = _cases(seed=4, count=12)
    for c in cases:
        for k in ('g', 's'):
            c.views[k].zero_()
    gs = dict(GS0, d_numerator=2e-9)
    mid, blk = _run(cases, gs=gs)
    assert float(blk[S['skip']]) == 1.0
    for k in ('d', 'd_max', 'd_hat', 'step'):
        assert float(blk[S[k]]) == gs[k], k
    assert float(blk[S['d_numerator']]) == 2e-9 * P._beta3(HYPER)
    assert all(torch.equal(_bits(c.views['p'].cpu()), _bits(c.before['p'].to(c.dtype))) for c in cases)


def test_the_specification_is_the_torch_op_text_on_cuda():
    """the recalled text as torch ops on CUDA tensors (where the reference trains), bf16 and fp32, two groups, one
    parameter without a gradient at step 2: m, v, s and p bit-identical to the emulation given the text's own d"""
    shapes = [(7,), (64, 33), (3, 5, 7), (4097,), (17, 241), (), ((1 << 18) + 5,)]
    for dtype in (BF16, torch.float32):
        gen = torch.Generator().manual_seed(11)
        ps = [((torch.randn(s, generator=gen) * 0.05).to(dtype)).cuda() for s in shapes]
        targets = [(torch.randn(s, generator=gen) * 0.05).cuda() for s in shapes]
        groups = [dict(P.DEFAULTS, weight_decay=0.01, params=ps[:4]),
                  dict(P.DEFAULTS, weight_decay=0.0, fixed_decay=True, params=ps[4:])]
        groups[1]['weight_decay'] = 0.02
        states, gs = {}, P.init_group_state(1e-6)
        for step in range(5):
            grads, k = [], 0
            for g in groups:
                gl = []
                for p in g['params']:
                    grad = (p.float() - targets[k]) + torch.randn(p.shape, generator=gen).cuda() * 1e-3
                    gl.append(None if (step == 2 and k == 1) else grad.to(dtype))
                    k += 1
                grads.append(gl)
            sc = P.step_scalars(dict(gs, d_numerator=float(gs['d_numerator'])), groups[0])
            pre = [[p.cpu() for p in g['params']] for g in groups]
            pre_states = {i: {kk: vv.cpu() for kk, vv in st.items()} for i, st in states.items()}
            assert P.prodigy_step_torch_ops(groups, grads, states, gs)
            for gi, (g, gl) in enumerate(zip(groups, grads)):
                for pi, (p, grad) in enumerate(zip(g['params'], gl)):
                    if grad is None:
                        continue
                    st0 = pre_states.get(id(p)) or P.init_state(pre[gi][pi])
                    m, v, s, _, _ = P.prodigy_stats_emulated(pre[gi][pi], grad.cpu(), st0['p0'], st0['s'],
                                                             st0['exp_avg'], st0['exp_avg_sq'], sc)
                    pn = P.prodigy_apply_emulated(pre[gi][pi], m, v, d_lr=sc['d_lr'], d=gs['d'], eps=g['eps'],
                                                  weight_decay=g['weight_decay'], fixed_decay=g['fixed_decay'])
                    st = states[id(p)]
                    for name, a, b in (('m', m, st['exp_avg']), ('v', v, st['exp_avg_sq']), ('s', s, st['s']),
                                       ('p', pn, p)):
                        assert torch.equal(_bits(a), _bits(b.cpu())), (dtype, step, name, tuple(p.shape))


def test_a_whole_step_does_not_synchronise_nor_keep_gradients(monkeypatch):
    """three steps with fresh gradient tensors each (as the engine gives them) under sync-debug mode: the arguments
    are packed once, and no gradient outlives zero_grad(set_to_none=True)"""
    import gc
    import weakref
    from diffusion_pipe_b200 import ops, optim
    packs = []
    real_pack = ops.prodigy_pack
    monkeypatch.setattr(ops, 'prodigy_pack', lambda *a, **k: packs.append(1) or real_pack(*a, **k))
    gen = torch.Generator().manual_seed(1)
    ps = [torch.nn.Parameter((torch.randn(s, generator=gen) * 0.05).to(dt).cuda())
          for s, dt in (((64, 96), BF16), ((96,), BF16), ((3, 4, 5), torch.float32), ((7,), torch.float32))]
    opt = optim.Prodigy([{'params': ps[:3]}, {'params': ps[3:], 'weight_decay': 0.0}], weight_decay=0.01)
    grads = [[(torch.randn(p.shape, generator=gen) * 1e-2).to(p.dtype).cuda() for p in ps] for _ in range(3)]
    torch.cuda.synchronize()
    versions = [p._version for p in ps]
    for k in range(3):
        for p, g in zip(ps, grads[k]):
            p.grad = g
        del g                   # the loop variable would keep the last gradient alive
        torch.cuda.set_sync_debug_mode('error')
        try:
            opt.step()          # step 1: state creation and argument packing included
        finally:
            torch.cuda.set_sync_debug_mode(0)
        refs = [weakref.ref(g) for g in grads[k]]
        grads[k] = None
        opt.zero_grad(set_to_none=True)
        gc.collect()
        assert all(r() is None for r in refs)
    assert len(packs) == 1
    assert int(opt.param_groups[1]['step']) == 3
    assert all(p._version >= v + 3 for p, v in zip(ps, versions))


# ---------------------------------------------------------------------------------------------------------------------
# engine runs
# ---------------------------------------------------------------------------------------------------------------------
class _TorchOpsProdigy(torch.optim.Optimizer):
    """the recalled torch-op text (oracle/prodigy_ref.py prodigy_step_torch_ops) on the GPU, with the groups a Prodigy
    built by the factory has"""

    def __init__(self, like):
        groups = [{k: v for k, v in g.items() if k not in ('step', 'd', 'd_max', 'd_hat', 'd_numerator', 'd_denom')}
                  for g in like.param_groups]
        super().__init__(groups, {})
        self.gs = P.init_group_state(like.param_groups[0]['d0'])
        self.tstates = {}

    @torch.no_grad()
    def step(self, closure=None):
        P.prodigy_step_torch_ops(self.param_groups, [[p.grad for p in g['params']] for g in self.param_groups],
                                 self.tstates, self.gs)


def _flux():
    from test_flux_e2e_gpu import _batch, _make
    model, _ = _make(3)
    return model, lambda s: [_batch(1, 10 * s + i) for i in range(2)]


def _qwen_lora():
    from test_automagic_gpu import _qwen_lora as make
    return make()


def _engine(model, torch_ops=False):
    import train as T
    from diffusion_pipe_b200.pipe import ManualPipelineModule, initialize
    pm = ManualPipelineModule(layers=model.to_layers(), num_stages=1, partition_method='parameters',
                              manual_partition_split=None, loss_fn=model.get_loss_fn(), dynamic_shape=True)
    engine, _, _, _ = initialize(model=pm, config={'train_micro_batch_size_per_gpu': 1, 'gradient_accumulation_steps': 2,
                                                   'gradient_clipping': 1.0, 'steps_per_print': 0})
    params = [p for p in pm.parameters() if p.requires_grad]
    factory = T.make_optimizer_factory({'optimizer': {'type': 'Prodigy', 'lr': 1, 'weight_decay': 0.01}}, model)
    engine._configure_optimizer((lambda ps: _TorchOpsProdigy(factory(ps))) if torch_ops else factory, params)
    return engine, pm, params


@pytest.mark.parametrize('family', ['flux', 'qwen_lora'])
def test_engine_steps_against_the_torch_op_text_and_resume(family, tmp_path):
    make = {'flux': _flux, 'qwen_lora': _qwen_lora}[family]
    model, batches = make()
    init = {n: p.detach().clone() for n, p in model.transformer.named_parameters()}
    engine, pm, params = _engine(model)
    losses, ds = [], []
    for s in range(4):
        losses.append(float(engine.train_batch(iter(batches(s)))))
        ds.append(float(engine.optimizer.param_groups[0]['d']))
        if s == 2:
            engine.save_checkpoint(str(tmp_path))
    final = {n: p.detach().clone() for n, p in model.transformer.named_parameters()}

    model_t, _ = make()
    with torch.no_grad():
        for n, p in model_t.transformer.named_parameters():
            p.copy_(init[n])
    engine_t, _, _ = _engine(model_t, torch_ops=True)
    for s in range(4):
        lt = float(engine_t.train_batch(iter(batches(s))))
        dt = engine_t.optimizer.gs['d']
        assert abs(lt - losses[s]) <= 1e-3 * abs(losses[s]), (s, lt, losses[s])
        assert abs(dt - ds[s]) <= 1e-4 * ds[s], (s, dt, ds[s])

    model2, _ = make()
    with torch.no_grad():
        for n, p in model2.transformer.named_parameters():
            p.copy_(init[n])
    engine2, _, _ = _engine(model2)
    engine2.load_checkpoint(str(tmp_path))
    assert int(engine2.optimizer.param_groups[0]['step']) == 3
    assert float(engine2.optimizer.param_groups[0]['d']) == ds[2]
    engine2.train_batch(iter(batches(3)))
    assert float(engine2.optimizer.param_groups[0]['d']) == ds[3]
    for n, p in model2.transformer.named_parameters():
        assert torch.equal(_bits(p.detach()), _bits(final[n])), n
