"""GPU: the CAME step kernels (csrc/came.cu).  Over 160 mixed tensors (bf16 / fp32; 0-D, 1-D, 2-D, 4-D and LoRA factor
shapes; empty tensors; views 1-7 elements into guarded buffers, every fifth with exp_avg one element off the others'
offset mod 16 B) and three steps, one of them without clipping, two groups' lr and wd, one parameter without a
gradient: the fp64 sums within 1e-12 of fp64, weights and state bit-identical to oracle/came_ref.py fed with the
kernels' sums, guard bands untouched, two runs equal bit for bit; the emulation against the torch-op text on CUDA; no
host synchronisation in a whole CAME.step() and no gradient kept past it.  Then a small Flux model (full fine-tune) and
a small Qwen-Image LoRA model train 4 steps with `type = 'CAME'` through the engine against the torch-op text stepped in
a second engine, and resume from a checkpoint with the same bits."""
import os
import sys

import pytest
import torch

from oracle import came_ref as CR

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
GUARD = 16
SHAPES = [(1,), (7,), (4097,), ((1 << 20) + 3,), (), (17, 241), (32, 3072), (3072, 32), (3, 5, 7, 9), (8193,),
          (2, 8192), (300, 1000), (0,), (0, 5), (1, 1)]
STATE = ('m', 'row', 'col', 'res_row', 'res_col', 'v')
KEYS = {'m': 'exp_avg', 'row': 'exp_avg_sq_row', 'col': 'exp_avg_sq_col', 'res_row': 'exp_avg_res_row',
        'res_col': 'exp_avg_res_col', 'v': 'exp_avg_sq'}


def _bits(t):
    return t.view(torch.int16) if t.dtype == BF16 else t.view(torch.int32) if t.dtype == torch.float32 else t


def _guarded(x, dtype, off, gen):
    n = x.numel()
    buf = (torch.randn(off + n + GUARD, generator=gen) * 7).to(dtype).cuda()
    view = buf[off:off + n].view(x.shape)
    view.copy_(x.to(dtype))
    return buf, view


class Case:
    """one parameter with its gradient and state as guarded CUDA views"""

    def __init__(self, i, shape, dtype, gen):
        self.shape, self.dtype, self.i = shape, dtype, i
        self.fact = len(shape) >= 2
        st = CR.init_state(torch.zeros(shape))
        off = 1 + i % 7
        self.bufs = {}
        vals = {'p': torch.randn(shape, generator=gen) * 0.05, 'g': torch.randn(shape, generator=gen) * 1e-2,
                'm': torch.randn(shape, generator=gen) * 1e-3}
        if self.fact:
            for k in ('row', 'col', 'res_row', 'res_col'):
                vals[k] = torch.rand(st[KEYS[k]].shape, generator=gen) * 1e-4
        else:
            vals['v'] = torch.rand(shape, generator=gen) * 1e-4
        for k, x in vals.items():
            self.bufs[k] = _guarded(x, dtype, off + (1 if k == 'm' and i % 5 == 0 else 0), gen)
        self.views = {k: v for k, (_, v) in self.bufs.items()}
        self.guards0 = {k: b.cpu() for k, (b, _) in self.bufs.items()}

    def new_grad(self, gen):
        self.views['g'].copy_((torch.randn(self.shape, generator=gen) * 1e-2).to(self.dtype))

    def snapshot(self):
        return {k: v.cpu().clone() for k, v in self.views.items()}

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
    out = []
    for i in range(count):
        shape = SHAPES[i % len(SHAPES)]
        if i >= 2 * len(SHAPES) and torch.Size(shape).numel() >= (1 << 18):
            shape = (17, 241)
        out.append(Case(i, shape, (BF16, torch.float32)[(i // len(SHAPES)) % 2], gen))
    return out, gen


def _hyper(i):
    """two groups: even cases lr 1e-3 / wd 0.01, odd ones lr 3e-3 / wd 0 (every third fixed decay)"""
    return dict(lr=1e-3 if i % 2 == 0 else 3e-3, weight_decay=0.01 if i % 2 == 0 else 0.0, fixed_decay=i % 3 == 0,
                betas=(0.9, 0.999, 0.9999), eps1=1e-30, eps2=1e-16)


def _pack(cases):
    from diffusion_pipe_b200 import ops
    v = [c.views for c in cases]
    hs = [_hyper(c.i) for c in cases]
    return ops.came_pack([x['p'] for x in v], [x['m'] for x in v], *[[x.get(k) for x in v] for k in STATE[1:5]],
                         [x.get('v') for x in v], [h['weight_decay'] for h in hs], [h['betas'] for h in hs],
                         [h['eps1'] for h in hs], [h['eps2'] for h in hs], [h['fixed_decay'] for h in hs])


def _sums_dict(c, s):
    s = s.cpu()
    if not c.fact:
        return {'sumsq': s[:1]}
    L, R, C = CR.dims(c.shape)
    out, k = {'sumsq': s[:1]}, 1
    for pre in ('sq', 'res'):
        for name, n in (('_row', L * R), ('_col', L * C), ('_rm', L)):
            out[pre + name] = s[k:k + n]
            k += n
    return out


def test_kernels_match_the_specification_over_three_steps():
    cases, gen = _cases()
    assert len(cases) >= 150
    c5 = cases[5]
    before5 = None
    from diffusion_pipe_b200 import ops
    # step by step, so that the parameter without a gradient at step 2 can be checked to stay put
    for step, clip in enumerate((1.0, 1.0, 1e4)):
        if step == 1:
            before5 = {k: v for k, v in c5.snapshot().items() if k != 'g'}
        _run_steps_one(cases, gen, step, clip, ops)
        if step == 1:
            assert all(torch.equal(_bits(c5.views[k].cpu()), _bits(v)) for k, v in before5.items())
    assert all(c.guards_intact() for c in cases)


def _run_steps_one(cases, gen, step, clip, ops):
    sub = [c for c in cases if not (step == 1 and c.i == 5)]
    for c in cases:
        c.new_grad(gen)
    args = _pack(sub)
    before = [c.snapshot() for c in sub]
    ops.came_step(args, [c.views['g'] for c in sub], [_hyper(c.i)['lr'] for c in sub], clip)
    torch.cuda.synchronize()
    clipped = 0
    for j, (c, b) in enumerate(zip(sub, before)):
        if c.views['p'].numel() == 0:
            continue
        ksums = _sums_dict(c, args.sums[j])
        st = {KEYS[k]: b[k] for k in STATE if k in b}
        pn, new, own, cd = CR.came_param_emulated(b['p'], b['g'], st, clip_threshold=clip, sums=ksums, **_hyper(c.i))
        clipped += cd > 1.0
        for k, want in own.items():                                      # the kernels' sums against fp64
            got = ksums[k].double()
            assert float((got - want).abs().max()) <= 1e-12 * max(float(want.abs().max()), 1e-300), \
                (step, c.i, c.shape, k)
        assert torch.equal(_bits(c.views['p'].cpu()), _bits(pn)), (step, c.i, c.shape, c.dtype)
        for k in STATE:
            if k in c.views:
                assert torch.equal(_bits(c.views[k].cpu()), _bits(new[KEYS[k]])), (step, c.i, c.shape, k)
        assert float(args.fac[j][0]) == cd
    assert (clipped > 0) == (clip == 1.0), (step, clipped)


def test_two_runs_give_equal_bits():
    from diffusion_pipe_b200 import ops
    outs = []
    for _ in range(2):
        cases, gen = _cases(seed=8, count=60)
        for step in range(2):
            sub = cases
            for c in cases:
                c.new_grad(gen)
            args = _pack(sub)
            ops.came_step(args, [c.views['g'] for c in sub], [_hyper(c.i)['lr'] for c in sub], 1.0)
        torch.cuda.synchronize()
        outs.append([c.views[k].cpu() for c in cases for k in c.views] + [s.cpu() for s in args.sums])
    assert all(torch.equal(_bits(a), _bits(b)) for a, b in zip(*outs))


def test_the_specification_against_the_torch_op_text_on_cuda():
    """the recalled text as torch ops on CUDA tensors (where the reference trains), bf16 and fp32, two groups, one
    parameter without a gradient at step 2, three steps, the last without clipping: within the tolerance of
    tests/test_came_host_logic.py agree() (torch reduces in fp32 in its own order and takes an approximate rsqrt)"""
    from test_came_host_logic import STATE_KEYS, agree
    shapes = [(7,), (64, 33), (3, 5, 7), (4097,), (17, 241), (), (256, 1536), ((1 << 18) + 5,)]
    for dtype in (BF16, torch.float32):
        gen = torch.Generator().manual_seed(11)
        ps = [((torch.randn(s, generator=gen) * 0.05).to(dtype)).cuda() for s in shapes]
        groups = [dict(CR.DEFAULTS, lr=1e-3, weight_decay=0.01, params=ps[:4]),
                  dict(CR.DEFAULTS, lr=3e-3, weight_decay=0.02, fixed_decay=True, params=ps[4:])]
        emu = [dict(g, params=[p.cpu().clone() for p in g['params']]) for g in groups]
        ts, es = {}, {}
        for step, clip in enumerate((1.0, 1.0, 1e4)):
            grads = [[None if (step == 1 and gi == 0 and k == 1) else
                      (torch.randn(p.shape, generator=gen) * 1e-2).to(dtype).cuda() for k, p in enumerate(g['params'])]
                     for gi, g in enumerate(groups)]
            tb = [p.cpu() for g in groups for p in g['params']]
            eb = [p.clone() for g in emu for p in g['params']]
            CR.came_step_torch_ops(groups, grads, ts, clip)
            CR.came_step_emulated(emu, [[None if x is None else x.cpu() for x in gl] for gl in grads], es, clip)
            for k, (a, b, e0, p0) in enumerate(zip([p for g in emu for p in g['params']],
                                                   [p.cpu() for g in groups for p in g['params']], eb, tb)):
                da, db = a.float() - e0.float(), b.float() - p0.float()
                assert agree(da, db, dtype, db, p0), (dtype, step, k, tuple(a.shape))
            for pe, pt in zip([p for g in emu for p in g['params']], [p for g in groups for p in g['params']]):
                if id(pt) in ts:
                    for key in STATE_KEYS:
                        if key in ts[id(pt)]:
                            assert agree(es[id(pe)][key], ts[id(pt)][key].cpu(), dtype, ts[id(pt)][key].cpu()), \
                                (dtype, step, key, tuple(pt.shape))


def test_a_whole_step_does_not_synchronise_nor_keep_gradients(monkeypatch):
    """three steps with fresh gradient tensors each (as the engine gives them) under sync-debug mode: the arguments
    are packed once, lr changes reach the kernels, and no gradient outlives zero_grad(set_to_none=True)"""
    import gc
    import weakref
    from diffusion_pipe_b200 import ops, optim
    packs = []
    real_pack = ops.came_pack
    monkeypatch.setattr(ops, 'came_pack', lambda *a, **k: packs.append(1) or real_pack(*a, **k))
    gen = torch.Generator().manual_seed(1)
    ps = [torch.nn.Parameter((torch.randn(s, generator=gen) * 0.05).to(dt).cuda())
          for s, dt in (((64, 96), BF16), ((96,), BF16), ((3, 4, 5), torch.float32), ((7,), torch.float32))]
    opt = optim.CAME([{'params': ps[:3]}, {'params': ps[3:], 'weight_decay': 0.0}], lr=1e-3, weight_decay=0.01)
    grads = [[(torch.randn(p.shape, generator=gen) * 1e-2).to(p.dtype).cuda() for p in ps] for _ in range(3)]
    torch.cuda.synchronize()
    versions = [p._version for p in ps]
    for k in range(3):
        opt.param_groups[0]['lr'] = 1e-3 * (k + 1)
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
    assert float(opt._packed[1]._lr[0]) == 3e-3
    assert all(opt.state[p]['step'] == 3 for p in ps)
    assert all(p._version >= v + 3 for p, v in zip(ps, versions))


# ---------------------------------------------------------------------------------------------------------------------
# engine runs
# ---------------------------------------------------------------------------------------------------------------------
class _TorchOpsCAME(torch.optim.Optimizer):
    """the recalled torch-op text (oracle/came_ref.py came_step_torch_ops) on the GPU, with the groups a CAME built by
    the factory has"""

    def __init__(self, like):
        super().__init__([dict(g) for g in like.param_groups], {})
        self.clip = like.clip_threshold
        self.tstates = {}

    @torch.no_grad()
    def step(self, closure=None):
        CR.came_step_torch_ops(self.param_groups, [[p.grad for p in g['params']] for g in self.param_groups],
                               self.tstates, self.clip)


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
    factory = T.make_optimizer_factory({'optimizer': {'type': 'CAME', 'lr': 1e-4, 'weight_decay': 0.01}}, model)
    engine._configure_optimizer((lambda ps: _TorchOpsCAME(factory(ps))) if torch_ops else factory, params)
    return engine, pm, params


@pytest.mark.parametrize('family', ['flux', 'qwen_lora'])
def test_engine_steps_against_the_torch_op_text_and_resume(family, tmp_path):
    make = {'flux': _flux, 'qwen_lora': _qwen_lora}[family]
    model, batches = make()
    init = {n: p.detach().clone() for n, p in model.transformer.named_parameters()}
    engine, pm, params = _engine(model)
    losses = []
    for s in range(4):
        losses.append(float(engine.train_batch(iter(batches(s)))))
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
        assert abs(lt - losses[s]) <= 1e-3 * abs(losses[s]), (s, lt, losses[s])
    moved = [n for n in final if not torch.equal(final[n], init[n])]
    assert moved

    model2, _ = make()
    with torch.no_grad():
        for n, p in model2.transformer.named_parameters():
            p.copy_(init[n])
    engine2, _, _ = _engine(model2)
    engine2.load_checkpoint(str(tmp_path))
    engine2.train_batch(iter(batches(3)))
    for n, p in model2.transformer.named_parameters():
        assert torch.equal(_bits(p.detach()), _bits(final[n])), n
