"""CPU: the Prodigy optimizer (`type = 'Prodigy'`) — the kernels' specification (oracle/prodigy_ref.py emulation)
against the recalled torch-op text, d's growth rules on a convex quadratic, the all-zero-gradient step, the optimizer
factory and constructor rules, the state dict and resume (with `ops.prodigy_*` replaced by an emulation-backed double
defined in this file), `train/prodigy_d` in a CLI run on the kernel doubles, and the C entry points' argument checks."""
import copy
import ctypes
import json
import os
import subprocess
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (ROOT, HERE):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from oracle import prodigy_ref as P  # noqa: E402

BF16 = torch.bfloat16
SHAPES = [(7,), (64, 33), (3, 5, 7), (1000,), (17, 241), ()]


def _bits(t):
    return t.view(torch.int16) if t.dtype == BF16 else t.view(torch.int32) if t.dtype == torch.float32 else t


@pytest.fixture
def one_thread():
    n = torch.get_num_threads()
    torch.set_num_threads(1)
    yield
    torch.set_num_threads(n)


def _groups(dtype, seed=0, wd=0.01):
    gen = torch.Generator().manual_seed(seed)
    ps = [(torch.randn(s, generator=gen) * 0.05).to(dtype) for s in SHAPES]
    targets = [(torch.randn(s, generator=gen) * 0.05).to(dtype) for s in SHAPES]
    return ([dict(P.DEFAULTS, weight_decay=wd, params=ps[:4]), dict(P.DEFAULTS, weight_decay=0.0, params=ps[4:])],
            targets, gen)


def _quadratic_grads(groups, targets, gen, step, drop=None):
    """gradients of sum (p - target)^2 / 2 plus noise; parameter `drop` gets none"""
    out, k = [], 0
    for g in groups:
        gl = []
        for p in g['params']:
            t = targets[k]
            grad = (p.float() - t.float()) + torch.randn(p.shape, generator=gen) * 1e-3
            gl.append(None if k == drop else grad.to(p.dtype))
            k += 1
        out.append(gl)
    return out


def _ulps(a, b, dtype, ref=None):
    """|a - b| in units of the last place in dtype of ref (default b)"""
    ref = b if ref is None else ref
    e = torch.floor(torch.log2(ref.double().abs().clamp_min(2.0 ** -126)))
    return (a.double() - b.double()).abs() / torch.pow(2.0, e - (7 if dtype == BF16 else 23))


@pytest.mark.parametrize('dtype', [torch.float32, BF16])
def test_emulation_agrees_with_the_torch_op_text(dtype, one_thread):
    """From the same state each step, given the text's new d.  The specification follows torch's CUDA kernels (bit for
    bit there: tests/test_prodigy_gpu.py); torch's CPU kernels evaluate addcmul and addcdiv in another order and round a
    bf16 add's alpha to bf16, so here: fp32 m and s bit for bit, v and p within two ulps (one rounding placed
    differently, measured in the ulp of the text's value, for p of the largest of it, the old p and the update); bf16
    within one ulp except where the rounded alpha's term cancels most of a sum (at most 1 % of the elements).  Over six steps with one
    parameter missing its gradient at step 2, d of the emulation within 1e-6 of the text's (fp32; bf16: the text rounds
    every tensor's dot and sum to bf16)."""
    groups, targets, gen = _groups(dtype)
    emu_groups = copy.deepcopy(groups)
    states, gs = {}, P.init_group_state(1e-6)
    emu_states, egs = {}, P.init_group_state(1e-6)
    far = total = 0
    for step in range(6):
        grads = _quadratic_grads(groups, targets, gen, step, drop=1 if step == 2 else None)
        sc = P.step_scalars(dict(gs, d_numerator=float(gs['d_numerator'])), groups[0])
        pre = [[p.clone() for p in g['params']] for g in groups]
        pre_states = {k: {kk: vv.clone() for kk, vv in v.items()} for k, v in states.items()}
        assert P.prodigy_step_torch_ops(groups, grads, states, gs)
        for gi, (g, gl) in enumerate(zip(groups, grads)):
            for pi, (p, grad) in enumerate(zip(g['params'], gl)):
                if grad is None:
                    continue
                st0 = pre_states.get(id(p)) or P.init_state(pre[gi][pi])
                m, v, s, _, _ = P.prodigy_stats_emulated(pre[gi][pi], grad, st0['p0'], st0['s'], st0['exp_avg'],
                                                         st0['exp_avg_sq'], sc)
                pn = P.prodigy_apply_emulated(pre[gi][pi], m, v, d_lr=sc['d_lr'], d=gs['d'], eps=g['eps'],
                                              weight_decay=g['weight_decay'], fixed_decay=g['fixed_decay'])
                st = states[id(p)]
                for name, a, b in (('m', m, st['exp_avg']), ('v', v, st['exp_avg_sq']), ('s', s, st['s']),
                                   ('p', pn, p)):
                    if dtype == torch.float32 and name in ('m', 's'):
                        assert torch.equal(_bits(a), _bits(b)), (step, name, tuple(p.shape))
                    elif dtype == torch.float32:
                        q = pre[gi][pi]
                        ref = torch.maximum(torch.maximum(b.abs(), q.abs()), (b - q).abs()) if name == 'p' else b
                        assert bool((_ulps(a, b, dtype, ref) <= 2).all()), (step, name, tuple(p.shape))
                    else:
                        far += int((_ulps(a, b, dtype) > 1).sum())
                        total += a.numel()
        P.prodigy_step_emulated(emu_groups, grads, emu_states, egs)
        assert egs['step'] == gs['step'] == step + 1
        tol = 1e-6 if dtype == torch.float32 else 2e-2
        assert abs(egs['d'] - gs['d']) <= tol * gs['d'], (step, egs['d'], gs['d'])
        assert abs(egs['d_max'] - gs['d_max']) <= tol * gs['d_max']
    if dtype == torch.float32:
        assert gs['d'] > 1e-6                               # d grew from d0 (bf16 weights near 0.05 do not move yet)
    else:
        assert far <= 0.01 * total, (far, total)


def test_fma_rounds_once():
    """the specification's fp32 fma rounds once, also where the fp64 sum falls exactly half-way between two fp32
    values: (1 + 2^-23) + (2^-12 (1 + 2^-15)) (2^-12 (1 - 2^-15)) = 1 + 2^-23 + 2^-24 - 2^-54 rounds down to 1 + 2^-23,
    while rounding through fp64 lands on the midpoint and ties to 1 + 2^-22"""
    a = torch.tensor([2.0 ** -12 * (1 + 2.0 ** -15), -(2.0 ** -12 * (1 + 2.0 ** -15)), 3.0])
    b = torch.tensor([2.0 ** -12 * (1 - 2.0 ** -15)] * 2 + [5.0])
    c = torch.tensor([1 + 2.0 ** -23, -(1 + 2.0 ** -23), 7.0])
    via_fp64 = (a.double() * b.double() + c.double()).float()
    assert via_fp64[0].item() == 1 + 2.0 ** -22                   # the double rounding the emulation avoids
    assert P._fma(a, b, c).tolist() == [1 + 2.0 ** -23, -(1 + 2.0 ** -23), 22.0]


def test_d_on_a_convex_quadratic(one_thread):
    """lr = 1: d never decreases, never exceeds d_max nor d_prev * growth_rate, grows from d0; the loss falls"""
    for growth in (float('inf'), 1.5):
        gen = torch.Generator().manual_seed(3)
        target = torch.randn(4096, generator=gen)
        p = torch.zeros(4096)
        groups = [dict(P.DEFAULTS, growth_rate=growth, params=[p])]
        states, gs = {}, P.init_group_state(1e-6)
        losses, prev = [], gs['d']
        for _ in range(60):
            losses.append(float(((p - target) ** 2).sum() / 2))
            P.prodigy_step_emulated(groups, [[(p - target).clone()]], states, gs)
            assert prev <= gs['d'] <= gs['d_max']
            assert prev == 1e-6 or gs['d'] <= prev * growth * (1 + 1e-15)      # d == d0 takes d_hat at once
            prev = gs['d']
        assert gs['d'] > 1e3 * 1e-6 and losses[-1] < 0.5 * losses[0], (gs['d'], losses[0], losses[-1])


@pytest.mark.parametrize('impl', ['torch_ops', 'emulated'])
def test_a_step_with_d_denom_zero_moves_the_statistics_only(impl):
    """every gradient zero and s zero (here: s cleared by hand after three steps): m, v and d_numerator decay as in any
    step; the weights, d, d_max, d_hat and the step count stay; the next real step is step 4"""
    groups, targets, gen = _groups(torch.float32)
    step = {'torch_ops': P.prodigy_step_torch_ops, 'emulated': P.prodigy_step_emulated}[impl]
    states, gs = {}, P.init_group_state(1e-6)
    for s in range(3):
        step(groups, _quadratic_grads(groups, targets, gen, s), states, gs)
    for st in states.values():
        st['s'].zero_()
    before = [p.clone() for g in groups for p in g['params']]
    st_before = {k: {kk: vv.clone() for kk, vv in v.items()} for k, v in states.items()}
    gs_before = {k: (float(v) if torch.is_tensor(v) else v) for k, v in gs.items()}
    assert gs_before['d_numerator'] != 0.0
    step(groups, [[torch.zeros_like(p) for p in g['params']] for g in groups], states, gs)
    assert all(torch.equal(a, b) for a, b in zip(before, [p for g in groups for p in g['params']]))
    for k in ('step', 'd', 'd_max', 'd_hat'):
        assert gs[k] == gs_before[k], k
    beta3 = P.DEFAULTS['betas'][1] ** 0.5
    assert abs(float(gs['d_numerator']) - beta3 * gs_before['d_numerator']) <= 1e-6 * abs(gs_before['d_numerator'])
    for k, st in states.items():
        assert torch.equal(st['exp_avg'], st_before[k]['exp_avg'] * P.f32(0.9))
        assert torch.equal(st['exp_avg_sq'], st_before[k]['exp_avg_sq'] * P.f32(0.999))
        assert not st['s'].any()
    step(groups, _quadratic_grads(groups, targets, gen, 4), states, gs)
    assert gs['step'] == 4


# ---------------------------------------------------------------------------------------------------------------------
# the optimizer on CPU, with the kernels replaced by the emulation
# ---------------------------------------------------------------------------------------------------------------------
class _Args:
    """the test double of ops.ProdigyArgs: the packed tensors, no gradients"""
    packs = 0

    def __init__(self, params, s, p0, m, v, weight_decay, eps, fixed_decay, device=None):
        type(self).packs += 1
        self.params, self.s, self.p0, self.m, self.v = params, s, p0, m, v
        self.wd, self.eps, self.fixed = weight_decay, eps, fixed_decay


def _emu_stats(args, grads, state, *, lr, betas, beta3, d0, d_coef, growth_rate, bias_correction, safeguard_warmup):
    from diffusion_pipe_b200 import _abi
    S = _abi.PRODIGY_SLOTS
    h = dict(lr=lr, betas=betas, beta3=beta3, d0=d0, d_coef=d_coef, growth_rate=growth_rate,
             bias_correction=bias_correction, safeguard_warmup=safeguard_warmup)
    gs = {k: float(state[S[k]]) for k in ('d', 'd_max', 'd_hat', 'd_numerator', 'd_denom')}
    gs['step'] = int(state[S['step']])
    sc = P.step_scalars(gs, h)
    sums = []
    for i, p in enumerate(args.params):
        m, v, s, dot, a = P.prodigy_stats_emulated(p, grads[i], args.p0[i], args.s[i], args.m[i], args.v[i], sc)
        args.m[i].copy_(m)
        args.v[i].copy_(v)
        args.s[i].copy_(s)
        sums.append((dot, a))
    new, skipped = P.prodigy_fold(gs, h, sc, sums)
    for k in ('d', 'd_max', 'd_hat', 'd_numerator', 'd_denom', 'step'):
        state[S[k]] = new[k]
    state[S['d_lr']] = sc['d_lr']
    state[S['skip']] = float(skipped)


def _emu_apply(args, state):
    from diffusion_pipe_b200 import _abi
    S = _abi.PRODIGY_SLOTS
    if float(state[S['skip']]):
        return
    for i, p in enumerate(args.params):
        p.data.copy_(P.prodigy_apply_emulated(p, args.m[i], args.v[i], d_lr=float(state[S['d_lr']]),
                                              d=float(state[S['d']]), eps=args.eps[i], weight_decay=args.wd[i],
                                              fixed_decay=args.fixed[i]))


@pytest.fixture
def emu_ops(monkeypatch):
    from diffusion_pipe_b200 import ops
    monkeypatch.setattr(ops, 'prodigy_pack', _Args)
    monkeypatch.setattr(ops, 'prodigy_stats', _emu_stats)
    monkeypatch.setattr(ops, 'prodigy_apply', _emu_apply)


def _optimizer(weights, **kw):
    from diffusion_pipe_b200 import optim
    ps = [torch.nn.Parameter(w.clone()) for w in weights]
    opt = optim.Prodigy([{'params': ps[:3]}, {'params': ps[3:], 'weight_decay': 0.0}], weight_decay=0.01, **kw)
    return opt, ps


def _step(opt, ps, gen):
    for p in ps:
        p.grad = (p.detach().float() * 0.5 + torch.randn(p.shape, generator=gen) * 1e-2).to(p.dtype)
    opt.step()


def test_the_optimizer_follows_the_emulation_and_shares_one_d(emu_ops):
    gen = torch.Generator().manual_seed(0)
    ws = [(torch.randn(s, generator=gen) * 0.05).to(dt) for s, dt in zip(SHAPES, (BF16, torch.float32) * 3)]
    opt, ps = _optimizer(ws)
    groups = [dict(P.DEFAULTS, weight_decay=0.01, params=[w.clone() for w in ws[:3]]),
              dict(P.DEFAULTS, weight_decay=0.0, params=[w.clone() for w in ws[3:]])]
    states, gs = {}, P.init_group_state(1e-6)
    g1, g2 = torch.Generator().manual_seed(1), torch.Generator().manual_seed(1)
    for _ in range(4):
        _step(opt, ps, g1)
        grads = [[(p.float() * 0.5 + torch.randn(p.shape, generator=g2) * 1e-2).to(p.dtype) for p in g['params']]
                 for g in groups]
        P.prodigy_step_emulated(groups, grads, states, gs)
        want = [p for g in groups for p in g['params']]
        assert all(torch.equal(_bits(a.detach()), _bits(b)) for a, b in zip(ps, want))
        assert float(opt.param_groups[0]['d']) == float(opt.param_groups[1]['d']) == gs['d']
        assert int(opt.param_groups[1]['step']) == gs['step']
    assert float(opt.mean_d()) == gs['d'] > 1e-6


def test_gradients_are_not_kept_and_the_pack_is_reused(emu_ops):
    """as in the engine, every step gets fresh gradient tensors and zero_grad(set_to_none=True) drops them: the
    optimizer keeps no reference to a gradient past step(), and the packed arguments are built once"""
    import gc
    import weakref
    gen = torch.Generator().manual_seed(4)
    ws = [(torch.randn(s, generator=gen) * 0.05).to(BF16) for s in SHAPES]
    opt, ps = _optimizer(ws)
    _Args.packs = 0
    for _ in range(3):
        _step(opt, ps, gen)
        refs = [weakref.ref(p.grad) for p in ps]
        opt.zero_grad(set_to_none=True)
        gc.collect()
        assert all(r() is None for r in refs)
    assert _Args.packs == 1
    ps[2].grad = None                                       # another set of parameters with gradients: packed anew
    for p in ps[:2] + ps[3:]:
        p.grad = torch.zeros_like(p)
    opt.step()
    assert _Args.packs == 2


def test_state_dict_round_trip_resume_and_float_scalars(emu_ops):
    gen = torch.Generator().manual_seed(2)
    ws = [(torch.randn(s, generator=gen) * 0.05).to(BF16) for s in SHAPES]
    opt, ps = _optimizer(ws)
    g = torch.Generator().manual_seed(7)
    for _ in range(3):
        _step(opt, ps, g)
    sd = opt.state_dict()
    for grp in sd['param_groups']:
        assert isinstance(grp['step'], int) and grp['step'] == 3
        for k in ('d', 'd_max', 'd_hat', 'd_numerator', 'd_denom'):
            assert isinstance(grp[k], float), k
    assert set(sd['state'][0]) == {'s', 'p0', 'exp_avg', 'exp_avg_sq'}
    opt2, ps2 = _optimizer([p.detach() for p in ps])
    opt2.load_state_dict(copy.deepcopy(sd))
    opt3, ps3 = _optimizer([p.detach() for p in ps])            # tensors instead of numbers load too
    sd3 = copy.deepcopy(sd)
    for grp in sd3['param_groups']:
        for k in ('d', 'd_max', 'd_hat', 'd_numerator', 'd_denom', 'step'):
            grp[k] = torch.tensor(float(grp[k]), dtype=torch.float64)
    opt3.load_state_dict(sd3)
    gens = [torch.Generator().manual_seed(9) for _ in range(3)]
    for _ in range(2):
        for o, q, gg in ((opt, ps, gens[0]), (opt2, ps2, gens[1]), (opt3, ps3, gens[2])):
            _step(o, q, gg)
    for q in (ps2, ps3):
        assert all(torch.equal(_bits(a.detach()), _bits(b.detach())) for a, b in zip(ps, q))
    assert float(opt2.param_groups[0]['d']) == float(opt.param_groups[0]['d'])


# ---------------------------------------------------------------------------------------------------------------------
# factory and constructor rules
# ---------------------------------------------------------------------------------------------------------------------
class _Model:
    def get_param_groups(self, params):
        return [{'params': params}]


@pytest.mark.parametrize('typ', ['Prodigy', 'prodigy'])
def test_factory_builds_prodigy_with_the_wd_split(typ):
    import train as T
    from diffusion_pipe_b200 import optim
    ps = [torch.nn.Parameter(torch.zeros(4, 6, dtype=BF16)), torch.nn.Parameter(torch.zeros(6, dtype=BF16))]
    opt = T.make_optimizer_factory({'optimizer': {'type': typ, 'lr': 1, 'weight_decay': 0.01}}, _Model())(ps)
    assert isinstance(opt, optim.Prodigy)
    g0, g1 = opt.param_groups
    for k, v in P.DEFAULTS.items():
        if k not in ('lr', 'weight_decay'):
            assert g0[k] == v and g1[k] == v, k
    assert (g0['lr'], g0['weight_decay'], g1['weight_decay']) == (1, 0.01, 0)
    assert g0['d'] is not g1['d'] and g0['d'].data_ptr() == g1['d'].data_ptr()       # one d for both groups
    assert float(g0['d']) == 1e-6 and int(g0['step']) == 0
    opt = T.make_optimizer_factory({'optimizer': {'type': typ, 'betas': [0.9, 0.99], 'beta2_half_life': 50}},
                                   _Model(), global_batch_size=5)(ps)
    assert opt.param_groups[0]['betas'] == (0.9, 0.5 ** (5 / 50))


def test_refused_options_and_unknown_kwargs():
    import train as T
    from diffusion_pipe_b200 import optim
    p = torch.nn.Parameter(torch.zeros(4, 4, dtype=BF16))
    with pytest.raises(TypeError):
        optim.Prodigy([p], not_an_option=1)
    with pytest.raises(NotImplementedError):
        optim.Prodigy([p], weight_decouple=False)
    with pytest.raises(NotImplementedError):
        T.make_optimizer_factory({'optimizer': {'type': 'Prodigy', 'gradient_release': True}}, _Model())([p])
    for dt in (torch.float16, torch.float8_e4m3fn):
        with pytest.raises(TypeError):
            optim.Prodigy([torch.nn.Parameter(torch.zeros(4, 4).to(dt), requires_grad=False)])
    opt = optim.Prodigy([p])
    p.grad = torch.ones(4, 4, dtype=BF16)
    with pytest.raises(TypeError, match='CUDA'):
        opt.step()
    for typ in ('adamw8bitkahan', 'stableadamw'):
        with pytest.raises(NotImplementedError):
            T.make_optimizer_factory({'optimizer': {'type': typ, 'lr': 1e-4}}, _Model())([p])


def test_cli_run_logs_prodigy_d(tmp_path, monkeypatch, emu_ops):
    """train.py on a small Flux model with the kernel doubles: metrics.jsonl carries train/prodigy_d with every loss"""
    import kernel_doubles
    import train as T
    from diffusion_pipe_b200 import ops
    kernel_doubles.install(monkeypatch, ops)
    ds = tmp_path / 'ds.toml'
    ds.write_text("[synthetic]\nnum_examples = 8\nresolution = 128\ntext_len = 32\nt5_dim = 64\nclip_dim = 32\n")
    cfgp = tmp_path / 'cfg.toml'
    cfgp.write_text(f"""
output_dir = '{tmp_path}/runs'
dataset = '{ds}'
epochs = 1
micro_batch_size_per_gpu = 1
gradient_accumulation_steps = 2
save_every_n_steps = 2
max_steps = 3
eval_before_first_step = false
[model]
type = 'flux'
dtype = 'bfloat16'
device = 'cpu'
transformer_config = {{ num_attention_heads = 2, num_layers = 1, num_single_layers = 1, joint_attention_dim = 64, pooled_projection_dim = 32 }}
[optimizer]
type = 'Prodigy'
lr = 1
weight_decay = 0.01
""")
    run_dir = T.main(['--config', str(cfgp)])
    lines = [json.loads(line) for line in open(os.path.join(run_dir, 'metrics.jsonl'))]
    ds_ = [line for line in lines if line['tag'] == 'train/prodigy_d']
    assert [line['x'] for line in ds_] == [1, 2, 3]
    assert ds_[0]['value'] == pytest.approx(1e-6) and all(line['value'] >= 1e-6 * (1 - 1e-6) for line in ds_)


# ---------------------------------------------------------------------------------------------------------------------
# C ABI
# ---------------------------------------------------------------------------------------------------------------------
def test_abi_structs_match_the_c_compiler(tmp_path):
    from diffusion_pipe_b200 import _abi
    pairs = (('dpipe_prodigy_tensor', _abi.ProdigyTensor), ('dpipe_prodigy_scalars', _abi.ProdigyScalars))
    src = '#include <stdio.h>\n#include <stddef.h>\n#include "dpipe.h"\nint main(void){\n'
    for name, cls in pairs:
        for f, _ in cls._fields_:
            src += f'  printf("{name} {f} %zu\\n", offsetof({name}, {f}));\n'
        src += f'  printf("{name} __size__ %zu\\n", sizeof({name}));\n'
    for k, v in _abi.PRODIGY_SLOTS.items():
        src += f'  printf("slot {k} %d\\n", DPIPE_PRODIGY_{k.upper()});\n'
    src += '  printf("slot __n__ %d\\n", DPIPE_PRODIGY_STATE_DOUBLES);\n  return 0; }\n'
    (tmp_path / 'off.c').write_text(src)
    subprocess.run(['gcc', '-std=c99', '-I', os.path.join(ROOT, 'include'), str(tmp_path / 'off.c'), '-o',
                    str(tmp_path / 'off')], check=True)
    out = subprocess.run([str(tmp_path / 'off')], check=True, capture_output=True, text=True).stdout.split()
    got = {(out[i], out[i + 1]): int(out[i + 2]) for i in range(0, len(out), 3)}
    for name, cls in pairs:
        for f, _ in cls._fields_:
            assert getattr(cls, f).offset == got[(name, f)], (name, f)
        assert ctypes.sizeof(cls) == got[(name, '__size__')]
    assert all(got[('slot', k)] == v for k, v in _abi.PRODIGY_SLOTS.items())
    assert got[('slot', '__n__')] == _abi.PRODIGY_STATE_DOUBLES


def _lib_or_skip():
    from diffusion_pipe_b200 import _lib
    try:
        return _lib.lib()
    except Exception as e:                                            # noqa: BLE001
        pytest.skip(f'native library not loadable here: {e}')


def test_entry_points_reject_bad_arguments_before_any_cuda_call():
    from diffusion_pipe_b200 import _abi
    lib = _lib_or_skip()
    t = (_abi.ProdigyTensor * 1)()
    for f in ('p', 'g', 'p0', 's', 'm', 'v'):
        setattr(t[0], f, ctypes.c_void_p(16))
    t[0].numel, t[0].dtype = 12, 0
    sc = _abi.ProdigyScalars(1.0, 0.9, 0.999, 0.9995, 1e-6, 1.0, float('inf'), 0, 0)
    blk, scratch = ctypes.c_void_p(64), ctypes.c_void_p(128)

    def rc(a, s=sc, state=blk, scr=scratch, n=1):
        return (lib.dpipe_prodigy_stats(a, n, ctypes.byref(s) if s is not None else None, state, scr, 1 << 20, None),
                lib.dpipe_prodigy_apply(a, n, state, None))
    for bad in (dict(dtype=2), dict(numel=-1), dict(g=None), dict(v=None), dict(p0=ctypes.c_void_p(17))):
        a = (_abi.ProdigyTensor * 1)()
        ctypes.memmove(a, t, ctypes.sizeof(t))
        for k, v in bad.items():
            setattr(a[0], k, v)
        assert all(r < 0 for r in rc(a)), bad
    assert all(r < 0 for r in rc(t, n=-1))
    assert rc(t, state=None)[0] < 0 and rc(t, state=None)[1] < 0
    assert rc(t, s=None)[0] < 0
    assert rc(t, s=_abi.ProdigyScalars(1.0, 0.9, 0.999, 0.9995, 0.0, 1.0, 1.0, 0, 0))[0] < 0
    assert lib.dpipe_prodigy_stats(t, 1, ctypes.byref(sc), blk, scratch, 3, None) < 0     # scratch too small
    need = ctypes.c_int64()
    assert lib.dpipe_prodigy_scratch_doubles(t, 1, ctypes.byref(need)) == 0 and need.value == 2 + 2
