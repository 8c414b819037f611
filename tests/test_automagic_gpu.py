"""GPU: the Automagic step kernels (csrc/automagic.cu).  Over ~150 mixed tensors in one call (bf16 / fp32, 1-D to 5-D,
sizes 1 to 2^20 + 3, views 1-7 elements into guarded buffers) at step 1 and at step 5: the statistics workspace against
fp64 on CPU, the apply phase bit-identical to oracle/automagic_ref.py automagic_apply_emulated fed with the kernels' own
workspace, the discrete state (lr codes, scale, polarity) bit-identical to the torch-op oracle, guard bands untouched,
two runs equal bit for bit, and no host synchronisation in a whole Automagic.step().  Then a small Flux model and a
small Qwen-Image LoRA model train 3 steps with `type = 'automagic'` through the engine, with those checks inside every
step, against the torch-op oracle stepped alongside, and resume from a checkpoint with the same bits."""
import copy
import os
import sys

import pytest
import torch

from oracle import automagic_ref as A

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
GUARD = 16
HYPER = dict(beta2=0.999, eps=1e-30, lr_bump=1e-6, min_lr=1e-7, max_lr=1e-3, clip_threshold=1.0, weight_decay=0.01)


def _bits(t):
    if t.dtype == BF16:
        return t.view(torch.int16)
    if t.dtype == torch.float32:
        return t.view(torch.int32)
    return t


def _guarded(vals, off, gen, dtype):
    """vals (CPU) copied into a CUDA buffer `off` elements in, with GUARD random elements after it"""
    n = vals.numel()
    if dtype in (torch.int8, torch.bool):
        buf = torch.randint(0, 2, (off + n + GUARD,), generator=gen).to(dtype).cuda()
    else:
        buf = (torch.randn(off + n + GUARD, generator=gen) * 7.0).to(dtype).cuda()
    view = buf[off:off + n].view(vals.shape)
    view.copy_(vals.to(dtype))
    return buf, view


SHAPES = [(1,), (7,), (4097,), ((1 << 20) + 3,), (), (1, 1), (7, 1), (1, 7), (17, 241), (241, 17), (32, 3072),
          (3072, 32), (1, 7, 1), (17, 1, 241, 1), (1, 17, 1, 1, 241), (3, 5, 7, 9), (2, 3, 4, 5, 6), (4097, 1)]


class Case:
    """one parameter with its state, as guarded CUDA views, and CPU copies of the pre-step values"""

    def __init__(self, shape, dtype, off, step, gen):
        self.shape, self.dtype, self.step = shape, dtype, step
        n = torch.Size(shape).numel()
        self.bufs = {}
        p = torch.randn(shape, generator=gen) * 0.05
        g = torch.randn(shape, generator=gen) * 1e-2
        if step == 1:
            codes = torch.full(shape, 127, dtype=torch.int8)
            pol = torch.zeros(shape, dtype=torch.bool)
            scale = A.f32(1e-6) / 127.0
            shift = torch.zeros(shape)
        else:
            codes = torch.randint(1, 128, shape, generator=gen).to(torch.int8)
            pol = torch.rand(shape, generator=gen) > 0.5
            scale = 3e-5 / 127.0
            shift = torch.randn(shape, generator=gen) * 1e-6
        for k, v, dt in (('p', p, dtype), ('g', g, dtype), ('code', codes, torch.int8), ('pol', pol, torch.bool),
                         ('shift', shift, BF16)):
            if k == 'shift' and dtype != BF16:
                continue
            self.bufs[k] = _guarded(v, off if k != 'code' else (off + 3) % 8, gen, dt)
        self.views = {k: v for k, (_, v) in self.bufs.items()}
        if len(shape) >= 2:
            rshape, cshape = shape[:-1], shape[:-2] + shape[-1:]
            z = step == 1
            self.row = (torch.zeros(rshape) if z else torch.rand(rshape, generator=gen) * 1e-4 + 1e-6).cuda()
            self.col = (torch.zeros(cshape) if z else torch.rand(cshape, generator=gen) * 1e-4 + 1e-6).cuda()
            self.v = None
        else:
            self.row = self.col = None
            self.v = (torch.zeros(shape) if step == 1 else torch.rand(shape, generator=gen) * 1e-4 + 1e-6).cuda()
        self.scale = torch.full((), scale, dtype=torch.float64, device='cuda')
        self.avg_lr = torch.zeros((), device='cuda')
        self.before = self.snapshot()
        self.guards0 = {k: b.cpu() for k, (b, _) in self.bufs.items()}

    def snapshot(self):
        s = {k: v.cpu().clone() for k, v in self.views.items()}
        for k in ('row', 'col', 'v'):
            t = getattr(self, k)
            s[k] = t.cpu().clone() if t is not None else None
        s['scale'] = float(self.scale.item())
        return s

    def round_bf16(self):
        return self.dtype == BF16 and self.step == 1

    def ref_state(self):
        """the pre-step state in the reference's format (bf16 statistics at step 1 of a bf16 parameter)"""
        b = self.before
        sdt = self.dtype if self.step == 1 else torch.float32
        st = {'step': self.step - 1, 'lr_mask': {'quantized': b['code'].clone(), 'scale': b['scale'],
                                                  'orig_dtype': torch.float32},
              'last_polarity': b['pol'].clone()}
        for k, name in (('row', 'exp_avg_sq_row'), ('col', 'exp_avg_sq_col'), ('v', 'exp_avg_sq')):
            if b[k] is not None:
                st[name] = b[k].to(sdt)
        if self.dtype == BF16:
            st['shift'] = b['shift'].clone()
        return st


def _args(cases, ws):
    return ([c.views['g'] for c in cases], [c.row for c in cases], [c.col for c in cases], [c.v for c in cases],
            [c.views['code'] for c in cases], [c.scale for c in cases], [c.views['pol'] for c in cases],
            [c.views.get('shift') for c in cases], [c.avg_lr for c in cases], ws, [c.round_bf16() for c in cases])


def _make_cases(step, seed=3, count=150):
    """count tensors cycling through SHAPES, bf16 and fp32 in alternate rounds; the two shapes of 2^20 + 3 elements
    only in the first two rounds (one bf16, one fp32)"""
    gen = torch.Generator().manual_seed(seed)
    small = [s for s in SHAPES if torch.Size(s).numel() < (1 << 20)]
    cases = []
    for i in range(count):
        shape = SHAPES[i % len(SHAPES)]
        if i >= 2 * len(SHAPES) and torch.Size(shape).numel() >= (1 << 20):
            shape = small[i % len(small)]
        dtype = (BF16, torch.float32)[(i // len(SHAPES)) % 2]
        cases.append(Case(shape, dtype, 1 + i % 7, step, gen))
    return cases


def _run(cases, hyper=HYPER):
    from diffusion_pipe_b200 import ops
    ps = [c.views['p'] for c in cases]
    ws = ops.automagic_workspace(ps)
    args = _args(cases, ws)
    ops.automagic_stats(ps, *args, **hyper)
    torch.cuda.synchronize()
    mid = [dict(ws=w.cpu().clone(), row=c.row.cpu().clone() if c.row is not None else None,
                col=c.col.cpu().clone() if c.col is not None else None,
                v=c.v.cpu().clone() if c.v is not None else None) for c, w in zip(cases, ws)]
    ops.automagic_apply(ps, *args, **hyper)
    torch.cuda.synchronize()
    return mid


def _rel(got, want):
    return ((got.double() - want).abs() / want.abs().clamp_min(1e-300)).max().item() if want.numel() else 0.0


@pytest.mark.parametrize('step', [1, 5])
def test_stats_apply_and_discrete_state(step):
    cases = _make_cases(step)
    mid = _run(cases)
    h = HYPER
    for c, m in zip(cases, mid):
        b = c.before
        tol = 2.0 ** -7 if c.round_bf16() else 1e-6
        g = b['g'].double()
        u0 = g * g + A.f32(h['eps'])
        ws = m['ws']
        L = 1
        for s in c.shape[:-2]:
            L *= s
        if len(c.shape) >= 2:
            R, C = c.shape[-2], c.shape[-1]
            row = h['beta2'] * b['row'].double() + (1 - h['beta2']) * u0.mean(-1)
            col = h['beta2'] * b['col'].double() + (1 - h['beta2']) * u0.mean(-2)
            assert _rel(m['row'], row) < tol and _rel(m['col'], col) < tol, (c.shape, c.dtype)
            rm = m['row'].double().reshape(L, R).mean(-1)
            assert _rel(ws[4:4 + L], rm) < tol
            rf = (m['row'].double().reshape(L, R) / ws[4:4 + L].double().unsqueeze(-1)).rsqrt()
            cf = m['col'].double().reshape(L, C).rsqrt()
            assert _rel(ws[4 + L:4 + L + L * R], rf.flatten()) < tol * 2
            assert _rel(ws[4 + L + L * R:], cf.flatten()) < tol * 2
            u = (ws[4 + L:4 + L + L * R].double().reshape(L, R, 1) * ws[4 + L + L * R:].double().reshape(L, 1, C)
                 * g.reshape(L, R, C)).reshape(c.shape)
        else:
            v = h['beta2'] * b['v'].double() + (1 - h['beta2']) * u0
            assert _rel(m['v'], v) < tol
            u = m['v'].double().rsqrt() * g
        rms = u.norm() / u.numel() ** 0.5
        clipdiv = max(rms.item() / h['clip_threshold'], 1.0)
        assert abs(ws[0].item() - clipdiv) <= tol * 4 * clipdiv, (c.shape, c.dtype, ws[0].item(), clipdiv)
        mask = b['code'].double() * A.f32(b['scale'])
        nl = torch.where((u > 0) == b['pol'], mask + h['lr_bump'], mask - h['lr_bump']).clamp(h['min_lr'], h['max_lr'])
        assert abs(ws[1].item() - nl.abs().max().item()) <= 1e-6 * nl.abs().max().item()
        assert abs(ws[2].item() - nl.mean().item()) <= 1e-6 * nl.mean().item()
        assert c.avg_lr.item() == ws[2].item()
        # apply: bit-identical to the emulation fed with the kernels' workspace
        kw = dict(rf=ws[4 + L:4 + L + L * R].reshape(c.shape[:-1]),
                  cf=ws[4 + L + L * R:].reshape(c.shape[:-2] + c.shape[-1:])) if len(c.shape) >= 2 else dict(v=m['v'])
        want = A.automagic_apply_emulated(b['p'], b['g'], codes=b['code'], polarity=b['pol'], shift=b.get('shift'),
                                          old_scale=float(ws[3]), new_scale=float(c.scale.item()),
                                          clipdiv=float(ws[0]), round_bf16=c.round_bf16(),
                                          weight_decay=h['weight_decay'], lr_bump=h['lr_bump'], min_lr=h['min_lr'],
                                          max_lr=h['max_lr'], **kw)
        got = (c.views['p'].cpu(), c.views['shift'].cpu() if 'shift' in c.views else None, c.views['code'].cpu(),
               c.views['pol'].cpu())
        for k, (w, x) in enumerate(zip(want, got)):
            if w is not None:
                assert torch.equal(_bits(w.to(x.dtype)), _bits(x)), (k, c.shape, c.dtype)
        assert float(ws[3]) == A.f32(b['scale'])
        # discrete state: equal to the torch-op oracle from the same pre-step state
        st = c.ref_state()
        A.automagic_step_torch_ops(b['p'].clone(), b['g'], st, beta2=h['beta2'], eps=(h['eps'], 1e-3),
                                   clip_threshold=h['clip_threshold'], weight_decay=h['weight_decay'],
                                   lr_bump=h['lr_bump'], min_lr=h['min_lr'], max_lr=h['max_lr'])
        assert torch.equal(st['lr_mask']['quantized'], got[2]), (c.shape, c.dtype)
        assert st['lr_mask']['scale'] == c.scale.item()
        assert torch.equal(st['last_polarity'], got[3])
        # guard bands
        for k, (buf, view) in c.bufs.items():
            off = (view.data_ptr() - buf.data_ptr()) // buf.element_size()
            n = view.numel()
            host, g0 = buf.cpu(), c.guards0[k]
            assert torch.equal(_bits(host[:off]), _bits(g0[:off])) and torch.equal(_bits(host[off + n:]),
                                                                                    _bits(g0[off + n:])), k


def test_two_runs_give_equal_bits():
    outs = []
    for _ in range(2):
        cases = _make_cases(5, seed=8, count=40)
        mid = _run(cases)
        outs.append([m['ws'] for m in mid] + [t for c in cases for t in (c.views['p'].cpu(), c.views['code'].cpu())]
                    + [c.row.cpu() for c in cases if c.row is not None])
    assert all(torch.equal(_bits(a), _bits(b)) for a, b in zip(*outs))


def test_a_whole_step_does_not_synchronise():
    from diffusion_pipe_b200 import optim
    gen = torch.Generator().manual_seed(1)
    ps = [torch.nn.Parameter((torch.randn(s, generator=gen) * 0.05).to(dt).cuda())
          for s, dt in (((64, 96), BF16), ((96,), BF16), ((3, 4, 5), torch.float32), ((7,), torch.float32))]
    opt = optim.Automagic([{'params': ps[:3]}, {'params': ps[3:], 'weight_decay': 0.0}], weight_decay=0.01)
    for p in ps:
        p.grad = torch.randn(p.shape, generator=gen).to(p.dtype).cuda() * 1e-2
    torch.cuda.synchronize()
    versions = [p._version for p in ps]
    torch.cuda.set_sync_debug_mode('error')
    try:
        opt.step()          # step 1: state creation included
        opt.step()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert all(opt.state[p]['step'] == 2 for p in ps)
    assert all(p._version >= v + 2 for p, v in zip(ps, versions))     # caches keyed on the version see new weights


# ---------------------------------------------------------------------------------------------------------------------
# engine runs
# ---------------------------------------------------------------------------------------------------------------------
def _flux():
    from test_flux_e2e_gpu import _batch, _make
    model, _ = _make(3)
    return model, lambda s: [_batch(1, 10 * s + i) for i in range(2)]


def _qwen_lora():
    from synth import fill_parameters
    from diffusion_pipe_b200.qwen_image import QwenImagePipeline
    from oracle import qwen_ref as Q
    cfg = {'num_attention_heads': 2, 'num_layers': 2, 'joint_attention_dim': 64}
    model = QwenImagePipeline({'model': {'dtype': 'bfloat16', 'transformer_config': cfg}})
    ref = fill_parameters(Q.RefQwenImageTransformer(dim=256, heads=2, num_layers=2, joint_dim=64))
    sd = ref.state_dict()
    with torch.no_grad():
        for n, p in model.transformer.named_parameters():
            p.copy_(sd[n].to(p.dtype))
    model.configure_adapter({'type': 'lora', 'rank': 8, 'alpha': 8, 'dropout': 0.0})
    with torch.no_grad():                                   # lora_B starts at zero: give it values so A gets gradients
        for n, p in model.transformer.named_parameters():
            if p.requires_grad and 'lora_B' in n:
                p.normal_(0, 0.02)

    def batches(s):
        out = []
        for i in range(2):
            g = torch.Generator().manual_seed(100 + 10 * s + i)
            latents, noise = torch.randn(1, 16, 1, 16, 24, generator=g), torch.randn(1, 16, 1, 16, 24, generator=g)
            pe = [torch.randn(12, 64, generator=g).bfloat16().float()]
            t = torch.sigmoid(torch.randn(1, generator=g))
            feats, (target, _) = Q.prepare_inputs(latents, pe, t, noise)
            out.append((feats, (target, torch.tensor([]))))
        return out
    return model, batches


def _engine(model):
    import train as T
    from diffusion_pipe_b200.pipe import ManualPipelineModule, initialize
    pm = ManualPipelineModule(layers=model.to_layers(), num_stages=1, partition_method='parameters',
                              manual_partition_split=None, loss_fn=model.get_loss_fn(), dynamic_shape=True)
    engine, _, _, _ = initialize(model=pm, config={'train_micro_batch_size_per_gpu': 1, 'gradient_accumulation_steps': 2,
                                                   'gradient_clipping': 1.0, 'steps_per_print': 0})
    params = [p for p in pm.parameters() if p.requires_grad]
    cfg = {'optimizer': {'type': 'automagic', 'weight_decay': 0.01}}
    engine._configure_optimizer(T.make_optimizer_factory(cfg, model), params)
    return engine, pm, params


def _ulp_bf16(x):
    e = torch.floor(torch.log2(x.abs().double().clamp_min(2.0 ** -126)))
    return torch.pow(2.0, e - 7)


@pytest.mark.parametrize('family', ['flux', 'qwen_lora'])
def test_engine_steps_checkpoint_and_oracle(family, tmp_path):
    from diffusion_pipe_b200 import ops
    make = {'flux': _flux, 'qwen_lora': _qwen_lora}[family]
    model, batches = make()
    init = {n: p.detach().clone() for n, p in model.transformer.named_parameters()}
    engine, pm, params = _engine(model)
    opt = engine.optimizer
    shadow = {id(p): [p.detach().cpu().clone(), None] for p in params}     # torch-op oracle stepped alongside
    real_stats, real_apply = ops.automagic_stats, ops.automagic_apply
    pending = {}
    checked = []

    def stats(ps, grads, rows, cols, vs, codes, scales, pols, shifts, avgs, ws, rnd, **h):
        pending['before'] = [dict(p=p.cpu(), g=g.cpu(), code=c.cpu(), pol=o.cpu(), scale=float(s.item()),
                                  shift=sh.cpu() if sh is not None else None) for p, g, c, o, s, sh in
                             zip(ps, grads, codes, pols, scales, shifts)]
        real_stats(ps, grads, rows, cols, vs, codes, scales, pols, shifts, avgs, ws, rnd, **h)

    def apply(ps, grads, rows, cols, vs, codes, scales, pols, shifts, avgs, ws, rnd, **h):
        wss = [w.cpu() for w in ws]
        vsc = [v.cpu() if v is not None else None for v in vs]
        real_apply(ps, grads, rows, cols, vs, codes, scales, pols, shifts, avgs, ws, rnd, **h)
        eps = h['eps']
        for i, (p, b) in enumerate(zip(ps, pending['before'])):
            w = wss[i]
            f, L, R, C = ops.automagic_dims(p.shape)
            kw = dict(rf=w[4 + L:4 + L + L * R].reshape(p.shape[:-1]),
                      cf=w[4 + L + L * R:].reshape(p.shape[:-2] + p.shape[-1:])) if f else dict(v=vsc[i])
            want = A.automagic_apply_emulated(b['p'], b['g'], codes=b['code'], polarity=b['pol'], shift=b['shift'],
                                              old_scale=float(w[3]), new_scale=float(scales[i].item()),
                                              clipdiv=float(w[0]), round_bf16=rnd[i],
                                              weight_decay=h['weight_decay'], lr_bump=h['lr_bump'],
                                              min_lr=h['min_lr'], max_lr=h['max_lr'], **kw)
            assert torch.equal(_bits(want[0].to(p.dtype)), _bits(p.cpu()))
            if want[1] is not None:
                assert torch.equal(_bits(want[1]), _bits(shifts[i].cpu()))
            # the torch-op oracle from the same pre-step state: identical discrete state
            sh = shadow[id(p)]
            if sh[1] is None:
                sh[1] = A.init_state(sh[0], opt.lr)
            ref = _ref_state_from(b, rows[i], cols[i], vs[i], rnd[i], sh[1], p.dtype)
            A.automagic_step_torch_ops(b['p'].clone(), b['g'], ref, beta2=h['beta2'], eps=(eps, 1e-3),
                                       clip_threshold=h['clip_threshold'], weight_decay=h['weight_decay'],
                                       lr_bump=h['lr_bump'], min_lr=h['min_lr'], max_lr=h['max_lr'])
            assert torch.equal(ref['lr_mask']['quantized'], codes[i].cpu()) and ref['lr_mask']['scale'] == scales[i].item()
            assert torch.equal(ref['last_polarity'], pols[i].cpu())
            # the shadow run: the torch-op oracle on its own state with the same gradients
            A.automagic_step_torch_ops(sh[0], b['g'], sh[1], beta2=h['beta2'], eps=(eps, 1e-3),
                                       clip_threshold=h['clip_threshold'], weight_decay=h['weight_decay'],
                                       lr_bump=h['lr_bump'], min_lr=h['min_lr'], max_lr=h['max_lr'])
        checked.append(len(ps))

    ops.automagic_stats, ops.automagic_apply = stats, apply
    try:
        for s in range(3):
            assert torch.isfinite(engine.train_batch(iter(batches(s))))
            if s == 1:
                engine.save_checkpoint(str(tmp_path))
    finally:
        ops.automagic_stats, ops.automagic_apply = real_stats, real_apply
    assert sum(checked) == 3 * len(params)
    eq = tot = 0
    for p in params:
        got, want = p.detach().cpu(), shadow[id(p)][0]
        same = _bits(got) == _bits(want)
        eq += int(same.sum())
        tot += got.numel()
        d = (got.double() - want.double()).abs()
        assert bool((d <= _ulp_bf16(want) + 0.0).all()) if got.dtype == BF16 else bool((d <= 1e-6).all())
    assert eq >= 0.999 * tot, (eq, tot)
    final = {n: p.detach().clone() for n, p in model.transformer.named_parameters()}

    # resume: a fresh engine, loaded after step 2, steps once to the same bits
    model2, _ = make()
    with torch.no_grad():
        for n, p in model2.transformer.named_parameters():
            p.copy_(init[n])
    engine2, pm2, params2 = _engine(model2)
    engine2.load_checkpoint(str(tmp_path))
    assert {st['step'] for st in engine2.optimizer.state.values()} <= {1, 2}
    engine2.train_batch(iter(batches(2)))
    for n, p in model2.transformer.named_parameters():
        assert torch.equal(_bits(p.detach()), _bits(final[n])), n


def _ref_state_from(b, row, col, v, rnd, shadow_state, dtype):
    """the kernels' pre-step state in the reference's format; its statistics come from the shadow oracle's state
    (pre-step), as the kernels' fp32 statistics hold their own reductions"""
    st = copy.deepcopy(shadow_state)
    st['lr_mask'] = {'quantized': b['code'].clone(), 'scale': b['scale'], 'orig_dtype': torch.float32}
    st['last_polarity'] = b['pol'].clone()
    if b['shift'] is not None:
        st['shift'] = b['shift'].clone()
    return st


def test_example_config_trains_saves_and_resumes(tmp_path):
    """examples/qwen_image_lora_automagic_synthetic.toml through train.py with a small transformer and dataset: two
    steps, a checkpoint, and a resumed third step that continues the Automagic state"""
    import json
    import train as T
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    text = open(os.path.join(root, 'examples', 'qwen_image_lora_automagic_synthetic.toml')).read()
    ds = tmp_path / 'ds.toml'
    ds.write_text("[synthetic]\nmodel = 'qwen_image'\nnum_examples = 8\nresolution = 128\ntext_len = 16\ntext_dim = 64\n")
    text = (text.replace("output_dir = '/tmp/dpipe_runs/qwen_image_lora_automagic_synthetic'", f"output_dir = '{tmp_path}/runs'")
            .replace("dataset = 'examples/dataset_synthetic_qwen.toml'", f"dataset = '{ds}'")
            .replace('gradient_accumulation_steps = 4', 'gradient_accumulation_steps = 2')
            .replace('save_every_n_epochs = 1', 'save_every_n_steps = 2\nmax_steps = 2')
            .replace("lazy_layers = true", "lazy_layers = true\ntransformer_config = { num_attention_heads = 2, "
                     "num_layers = 2, joint_attention_dim = 64 }"))
    assert "type = 'automagic'" in text and "transformer_dtype = 'float8'" in text
    cfgp = tmp_path / 'cfg.toml'
    cfgp.write_text(text)
    run_dir = T.main(['--config', str(cfgp)])
    assert os.path.exists(os.path.join(run_dir, 'latest'))
    cfgp.write_text(text.replace('max_steps = 2', 'max_steps = 3'))
    assert T.main(['--config', str(cfgp), '--resume_from_checkpoint']) == run_dir
    lines = [json.loads(line) for line in open(os.path.join(run_dir, 'metrics.jsonl'))]
    losses = [line for line in lines if line['tag'] == 'train/loss']
    assert [line['x'] for line in losses] == [1, 2, 3] and all(line['value'] == line['value'] for line in losses)
