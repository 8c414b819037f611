"""GPU: the AdamW8bit step kernel (csrc/adamw8bit.cu).  Over 160 mixed tensors in one call (bf16 / fp32; sizes below
4096 with fp32 states, 256·k, 256·k ± 1 and larger with 8-bit states; views 1-7 elements into guarded buffers, so
most are not 16-byte aligned; blocks with an all-zero gradient; a few non-finite gradient elements), three
consecutive steps: p, codes, absmax and fp32 states bit-identical to oracle/adamw8bit_ref.py, guard bands untouched;
two runs equal bit for bit; no host synchronisation in optim.AdamW8bit.step() and no gradient kept past it; the state
memory a first step allocates.  Then a small Flux model (full fine-tune) and a small Qwen-Image LoRA model train 4
steps with `type = 'AdamW8bit'` through the engine, every step checked against the emulation on that step's own
gradients, and resume from a checkpoint with the same bits."""
import os
import sys

import pytest
import torch

from oracle import adamw8bit_ref as A

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
GUARD = 16
SIZES = [1, 7, 255, 1000, 4095, 4096, 4097, 256 * 37, 256 * 37 + 1, 256 * 37 - 1, 65536 + 255, 300 * 256 + 129,
         (1 << 20) + 3]


def _bits(t):
    return t.view(torch.int16) if t.dtype == BF16 else t.view(torch.int32) if t.dtype == torch.float32 else t


def _guarded(x, off, gen, device='cuda'):
    """x copied into a CUDA buffer at element offset `off`, with random guard bands; returns (buffer, view)"""
    n = x.numel()
    if x.dtype == torch.uint8:
        buf = torch.randint(0, 256, (off + n + GUARD,), generator=gen, dtype=torch.uint8)
    else:
        buf = (torch.randn(off + n + GUARD, generator=gen) * 7).to(x.dtype)
    buf = buf.to(device)
    view = buf[off:off + n]
    view.copy_(x.reshape(-1))
    return buf, view


class Case:
    def __init__(self, i, n, dtype, gen):
        self.n, self.dtype = n, dtype
        q8 = n >= 4096
        g = torch.randn(n, generator=gen) * 1e-3
        if i % 6 == 1 and n >= 512:                              # an all-zero gradient block
            g[256:512] = 0.0
        if i % 17 == 3 and q8:                                   # non-finite gradient elements (8-bit path)
            g[5], g[n - 1] = float('inf'), float('nan')
        vals = {'p': (torch.randn(n, generator=gen) * 0.05).to(dtype), 'g': g.to(dtype)}
        if q8:
            nb = (n + 255) // 256
            vals.update(s1=torch.randint(0, 256, (n,), generator=gen, dtype=torch.uint8),
                        s2=torch.randint(0, 256, (n,), generator=gen, dtype=torch.uint8),
                        a1=torch.rand(nb, generator=gen) * 1e-3, a2=torch.rand(nb, generator=gen) * 1e-7)
            vals['a1'][0] = 0.0
        else:
            vals.update(s1=torch.randn(n, generator=gen) * 1e-3, s2=torch.rand(n, generator=gen) * 1e-7)
        off = i % 8                                              # p and g: 0-7 elements in (mostly not 16 B aligned)
        self.bufs = {k: _guarded(x, off if k in ('p', 'g') else (i % 3) * 3 if k in ('s1', 's2') else 0, gen)
                     for k, x in vals.items()}
        self.v = {k: v for k, (_, v) in self.bufs.items()}
        self.guards0 = {k: b.cpu() for k, (b, _) in self.bufs.items()}

    def state(self):
        return {k: self.v[k].cpu().clone() for k in self.v}

    def guards_intact(self):
        for k, (buf, view) in self.bufs.items():
            off = (view.data_ptr() - buf.data_ptr()) // buf.element_size()
            host, g0 = buf.cpu(), self.guards0[k]
            if not (torch.equal(_bits(host[:off]), _bits(g0[:off]))
                    and torch.equal(_bits(host[off + view.numel():]), _bits(g0[off + view.numel():]))):
                return False
        return True


def _cases(seed=3, count=160):
    gen = torch.Generator().manual_seed(seed)
    return [Case(i, SIZES[i % len(SIZES)] if i < 2 * len(SIZES) else SIZES[i % (len(SIZES) - 1)],
                 (BF16, torch.float32)[(i // len(SIZES)) % 2], gen) for i in range(count)]


HPS = [dict(lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2), dict(lr=3e-4, betas=(0.95, 0.99), eps=1e-6,
                                                                            weight_decay=0.0)]
QMAPS = (A.create_dynamic_map(True), A.create_dynamic_map(False))


def _scalars(cases, step):
    return [A.step_scalars(step=step, **HPS[i % 2]) for i in range(len(cases))]


def _run(cases, step):
    from diffusion_pipe_b200 import ops
    v = [c.v for c in cases]
    ops.adamw8bit_step([x['p'] for x in v], [x['g'] for x in v], [x['s1'] for x in v], [x['s2'] for x in v],
                       [x.get('a1') for x in v], [x.get('a2') for x in v], _scalars(cases, step),
                       QMAPS[0].cuda(), QMAPS[1].cuda())
    torch.cuda.synchronize()


def test_kernel_matches_the_specification_over_three_steps():
    cases = _cases()
    assert len(cases) > 64 and {c.n >= 4096 for c in cases} == {True, False}
    for step in (1, 2, 3):
        before = [c.state() for c in cases]
        _run(cases, step)
        for i, (c, b, sc) in enumerate(zip(cases, before, _scalars(cases, step))):
            want = A.adamw8bit_emulated(b['p'], b['g'], b['s1'], b['s2'], b.get('a1'), b.get('a2'), *QMAPS, **sc)
            got = (c.v['p'], c.v['s1'], c.v['s2'], c.v.get('a1'), c.v.get('a2'))
            for name, w, k in zip(('p', 'state1', 'state2', 'absmax1', 'absmax2'), want, got):
                if w is None:
                    assert k is None
                    continue
                assert torch.equal(_bits(k.cpu()), _bits(w.reshape(-1))), (step, i, name, c.n, c.dtype)
            assert c.guards_intact(), (step, i)
            if c.n >= 4096:
                assert bool(torch.isfinite(c.v['p'].float()).all())
            c.v['g'].copy_((torch.randn(c.n, generator=torch.Generator().manual_seed(step * 1000 + i)) * 1e-3)
                           .to(c.dtype))
            if i % 6 == 1 and c.n >= 512:
                c.v['g'][256:512] = 0.0


def test_two_runs_give_equal_bits():
    outs = []
    for _ in range(2):
        cases = _cases(seed=8, count=70)
        _run(cases, 1)
        _run(cases, 2)
        outs.append([c.v[k].cpu() for c in cases for k in c.v])
    assert all(torch.equal(_bits(a), _bits(b)) for a, b in zip(*outs))


def test_a_step_does_not_synchronise_nor_keep_gradients_and_allocates_its_state():
    """three steps with fresh gradient tensors each (as the engine gives them) under sync-debug mode; no gradient
    outlives zero_grad(set_to_none=True); the first step allocates exactly the state (each tensor rounded to the
    caching allocator's 512-byte granule): fp32 m, v below 4096 elements, else 2 B of codes + 8 B per 256 elements"""
    import gc
    import weakref
    from diffusion_pipe_b200 import optim
    gen = torch.Generator().manual_seed(1)
    shapes = (((64, 96), BF16), ((96,), BF16), ((3, 4, 5), torch.float32), ((3072, 513), BF16), ((10001,), torch.float32))
    ps = [torch.nn.Parameter((torch.randn(s, generator=gen) * 0.05).to(dt).cuda()) for s, dt in shapes]
    opt = optim.AdamW8bit([{'params': ps[:3]}, {'params': ps[3:], 'weight_decay': 0.0}])
    grads = [[(torch.randn(p.shape, generator=gen) * 1e-2).to(p.dtype).cuda() for p in ps] for _ in range(3)]

    def granule(nbytes):
        return (nbytes + 511) // 512 * 512
    want = 0
    for p in ps:
        n = p.numel()
        want += 2 * granule(4 * n) if n < 4096 else 2 * granule(n) + 2 * granule(4 * ((n + 255) // 256))
    torch.cuda.synchronize()
    versions = [p._version for p in ps]
    for k in range(3):
        for p, g in zip(ps, grads[k]):
            p.grad = g
        del g                   # the loop variable would keep the last gradient alive
        m0 = torch.cuda.memory_allocated()
        torch.cuda.set_sync_debug_mode('error')
        try:
            opt.step()          # step 1: state creation included
        finally:
            torch.cuda.set_sync_debug_mode(0)
        if k == 0:
            assert torch.cuda.memory_allocated() - m0 == want
        refs = [weakref.ref(g) for g in grads[k]]
        grads[k] = None
        opt.zero_grad(set_to_none=True)
        gc.collect()
        assert all(r() is None for r in refs)
    assert [opt.state[p]['step'] for p in ps] == [3] * 5
    assert all(p._version >= v + 3 for p, v in zip(ps, versions))


# ---------------------------------------------------------------------------------------------------------------------
# engine runs
# ---------------------------------------------------------------------------------------------------------------------
def _flux():
    from test_flux_e2e_gpu import _batch, _make
    model, _ = _make(3)
    return model, lambda s: [_batch(1, 10 * s + i) for i in range(2)]


def _qwen_lora():
    from test_automagic_gpu import _qwen_lora as make
    return make()


def _check_steps(opt, log):
    """step hooks: each step of `opt` against the emulation on the same weights, gradients and state"""
    snap = {}

    def pre(o, args, kwargs):
        snap.clear()
        for g in o.param_groups:
            for p in g['params']:
                if p.grad is not None:
                    st = o.state[p]
                    snap[p] = (p.detach().cpu().clone(), p.grad.cpu().clone(),
                               {k: (v.cpu().clone() if torch.is_tensor(v) else v) for k, v in st.items()}, g)

    def post(o, args, kwargs):
        oks = []
        for p, (w, grad, st, g) in snap.items():
            st = st if st else A.init_state(w, o.min_8bit_size)
            pn = A.step_emulated(w, grad, st, lr=g['lr'], betas=g['betas'], eps=g['eps'], weight_decay=g['weight_decay'])
            ok = torch.equal(_bits(pn), _bits(p.detach().cpu()))
            for k in ('state1', 'state2', 'absmax1', 'absmax2'):
                if k in st:
                    ok = ok and torch.equal(_bits(st[k]), _bits(o.state[p][k].cpu()))
            oks.append(ok)
        log.append(bool(oks) and all(oks))
    opt.register_step_pre_hook(pre)
    opt.register_step_post_hook(post)


def _engine(model, min_8bit_size, log=None):
    import train as T
    from diffusion_pipe_b200.pipe import ManualPipelineModule, initialize
    pm = ManualPipelineModule(layers=model.to_layers(), num_stages=1, partition_method='parameters',
                              manual_partition_split=None, loss_fn=model.get_loss_fn(), dynamic_shape=True)
    engine, _, _, _ = initialize(model=pm, config={'train_micro_batch_size_per_gpu': 1, 'gradient_accumulation_steps': 2,
                                                   'gradient_clipping': 1.0, 'steps_per_print': 0})
    params = [p for p in pm.parameters() if p.requires_grad]
    factory = T.make_optimizer_factory({'optimizer': {'type': 'AdamW8bit', 'lr': 1e-3, 'weight_decay': 0.01,
                                                      'min_8bit_size': min_8bit_size}}, model)

    def make(ps):
        opt = factory(ps)
        if log is not None:
            _check_steps(opt, log)
        return opt
    engine._configure_optimizer(make, params)
    return engine, pm, params


@pytest.mark.parametrize('family', ['flux', 'qwen_lora'])
def test_engine_steps_follow_the_emulation_and_resume(family, tmp_path):
    make = {'flux': _flux, 'qwen_lora': _qwen_lora}[family]
    min8 = 4096 if family == 'flux' else 1024              # the small model's LoRA factors: 2048 elements
    model, batches = make()
    init = {n: p.detach().clone() for n, p in model.transformer.named_parameters()}
    log = []
    engine, pm, params = _engine(model, min8, log)
    for s in range(4):
        loss = float(engine.train_batch(iter(batches(s))))
        assert loss == loss
        if s == 2:
            engine.save_checkpoint(str(tmp_path))
    assert len(log) == 4 and all(log), log
    opt = engine.optimizer
    kinds = {opt.state[p]['state1'].dtype for p in params}
    assert kinds == ({torch.uint8, torch.float32} if family == 'flux' else {torch.uint8}), kinds
    final = {n: p.detach().clone() for n, p in model.transformer.named_parameters()}

    model2, _ = make()
    with torch.no_grad():
        for n, p in model2.transformer.named_parameters():
            p.copy_(init[n])
    engine2, _, params2 = _engine(model2, min8)
    engine2.load_checkpoint(str(tmp_path))
    st2 = engine2.optimizer.state
    assert all(st2[p]['step'] == 3 for p in params2)
    assert {st2[p]['state1'].dtype for p in params2} == kinds
    assert all(st2[p]['absmax1'].dtype == torch.float32 for p in params2 if 'absmax1' in st2[p])
    engine2.train_batch(iter(batches(3)))
    for n, p in model2.transformer.named_parameters():
        assert torch.equal(_bits(p.detach()), _bits(final[n])), n
