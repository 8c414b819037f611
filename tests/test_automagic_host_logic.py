"""CPU: the Automagic optimizer (`type = 'automagic'`) — the torch-op oracle against the fixture recorded from the
reference's own code (tests/golden/automagic_golden.pt), the kernels' apply-phase specification against the torch-op
oracle, the optimizer factory and constructor rules, the state-dict format, loading a state dict written by the
reference and stepping on (with `ops.automagic_stats` / `ops.automagic_apply` replaced by an oracle-backed double
defined in this file), and the C entry points' argument checks."""
import ctypes
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

from oracle import automagic_ref as A  # noqa: E402

BF16 = torch.bfloat16
GOLDEN = os.path.join(HERE, 'golden', 'automagic_golden.pt')


def _bits(t):
    if t.dtype == BF16:
        return t.view(torch.int16)
    if t.dtype == torch.float32:
        return t.view(torch.int32)
    return t


def _ulp_bf16(x):
    e = torch.floor(torch.log2(x.abs().double().clamp_min(2.0 ** -126)))
    return torch.pow(2.0, e - 7)


@pytest.fixture
def one_thread():
    n = torch.get_num_threads()
    torch.set_num_threads(1)
    yield
    torch.set_num_threads(n)


@pytest.fixture(scope='module')
def golden():
    return torch.load(GOLDEN, weights_only=False)


def _hyper(cfg, grp):
    return dict(beta2=cfg.get('beta2', 0.999), eps=(1e-30, 1e-3), clip_threshold=cfg['clip_threshold'],
                weight_decay=cfg['weight_decay'] if grp == 0 else 0.0, lr_bump=cfg.get('lr_bump', 1e-6),
                min_lr=cfg.get('min_lr', 1e-7), max_lr=cfg.get('max_lr', 1e-3))


def _equal_state(mine, want):
    for k, v in want.items():
        if k == 'lr_mask':
            assert torch.equal(mine[k]['quantized'], v['quantized']) and mine[k]['scale'] == v['scale'], k
        elif torch.is_tensor(v):
            assert mine[k].dtype == v.dtype and torch.equal(_bits(mine[k]), _bits(v)), k
        else:
            assert mine[k] == v, k


def test_torch_op_oracle_equals_the_reference_fixture(golden, one_thread):
    for case, rec in golden['cases'].items():
        cfg = rec['config']
        lr = cfg['lr'] if cfg['lr'] <= 1e-3 else 1e-6
        ps, sts = [t.clone() for t in rec['init']], [None] * len(rec['init'])
        for s in range(golden['steps']):
            for i, (name, shape, grp) in enumerate(rec['params']):
                g = rec['grads'][s][i]
                if g is None:
                    continue
                sts[i] = sts[i] if sts[i] is not None else A.init_state(ps[i], lr)
                A.automagic_step_torch_ops(ps[i], g, sts[i], **_hyper(cfg, grp))
            for i in range(len(ps)):
                assert torch.equal(_bits(ps[i]), _bits(rec['weights'][s][i])), (case, s, i)
                if rec['states'][s][i] is not None:
                    _equal_state(sts[i], rec['states'][s][i])


def test_apply_emulation_fed_with_the_oracle_statistics_equals_the_oracle(golden, one_thread):
    """codes, scale and polarity exact; p and shift within one bf16 ulp on under 0.1 % of elements.  The one difference
    the fixture shows is at step 1 of a bf16 vector, where the statistics are bf16: torch's CPU bf16 rsqrt on the
    elements past the last full vector rounds 1/sqrt differently from the correctly rounded value (2032 instead of 2024
    for v = 2.44e-7), so u and then the shift differ by one bf16 ulp there."""
    diff = total = 0
    for case, rec in golden['cases'].items():
        cfg = rec['config']
        lr = cfg['lr'] if cfg['lr'] <= 1e-3 else 1e-6
        ps, sts = [t.clone() for t in rec['init']], [None] * len(rec['init'])
        for s in range(golden['steps']):
            for i, (name, shape, grp) in enumerate(rec['params']):
                g = rec['grads'][s][i]
                if g is None:
                    continue
                sts[i] = sts[i] if sts[i] is not None else A.init_state(ps[i], lr)
                h = _hyper(cfg, grp)
                p0, sh0 = ps[i].clone(), sts[i]['shift'].clone() if 'shift' in sts[i] else None
                rnd = ps[i].dtype == BF16 and sts[i]['step'] == 0
                stats = {}
                A.automagic_step_torch_ops(ps[i], g, sts[i], stats=stats, **h)
                got = A.automagic_apply_emulated(
                    p0, g, codes=stats['codes'], polarity=stats['polarity'], shift=sh0, old_scale=stats['old_scale'],
                    new_scale=stats['new_scale'], clipdiv=stats['clipdiv'], round_bf16=rnd,
                    weight_decay=h['weight_decay'], lr_bump=h['lr_bump'], min_lr=h['min_lr'], max_lr=h['max_lr'],
                    rf=stats.get('rf'), cf=stats.get('cf'), v=stats.get('v'))
                assert torch.equal(got[2], sts[i]['lr_mask']['quantized'])
                assert torch.equal(got[3], sts[i]['last_polarity'])
                pairs = [(got[0], ps[i])] + ([(got[1], sts[i]['shift'])] if got[1] is not None else [])
                for a, b in pairs:
                    ne = _bits(a) != _bits(b)
                    diff += int(ne.sum())
                    total += a.numel()
                    d = (a.double() - b.double()).abs()
                    tol = _ulp_bf16(b) if b.dtype == BF16 else b.abs().double() * 2.0 ** -23
                    assert bool((d <= tol).all()), (case, s, name)
    assert diff <= 1e-3 * total, (diff, total)


# ---------------------------------------------------------------------------------------------------------------------
# the optimizer on CPU, with the kernels replaced by the torch-op oracle
# ---------------------------------------------------------------------------------------------------------------------
def _oracle_stats(ps, grads, rows, cols, vs, codes, scales, pols, shifts, avgs, ws, rnd, *, beta2, eps, lr_bump,
                  min_lr, max_lr, clip_threshold, weight_decay):
    """the whole step through the torch-op oracle, written back into the optimizer's state tensors"""
    for i, p in enumerate(ps):
        sdt = p.dtype if rnd[i] else torch.float32
        st = {'step': 0 if rnd[i] else 1,
              'lr_mask': {'quantized': codes[i].clone(), 'scale': float(scales[i]), 'orig_dtype': torch.float32},
              'last_polarity': pols[i].clone(), 'avg_lr': avgs[i].clone()}
        if rows[i] is not None:
            st['exp_avg_sq_row'], st['exp_avg_sq_col'] = rows[i].to(sdt), cols[i].to(sdt)
        else:
            st['exp_avg_sq'] = vs[i].to(sdt)
        if shifts[i] is not None:
            st['shift'] = shifts[i]
        A.automagic_step_torch_ops(p.data, grads[i], st, beta2=beta2, eps=eps, clip_threshold=clip_threshold,
                                   weight_decay=weight_decay, lr_bump=lr_bump, min_lr=min_lr, max_lr=max_lr)
        if rows[i] is not None:
            rows[i].copy_(st['exp_avg_sq_row'])
            cols[i].copy_(st['exp_avg_sq_col'])
        else:
            vs[i].copy_(st['exp_avg_sq'])
        codes[i].copy_(st['lr_mask']['quantized'])
        scales[i].fill_(st['lr_mask']['scale'])
        pols[i].copy_(st['last_polarity'])
        avgs[i].copy_(st['avg_lr'])


def _oracle_apply(*args, **kw):
    pass


@pytest.fixture
def oracle_ops(monkeypatch):
    from diffusion_pipe_b200 import ops
    monkeypatch.setattr(ops, 'automagic_stats', _oracle_stats)
    monkeypatch.setattr(ops, 'automagic_apply', _oracle_apply)


def _fixture_optimizer(rec, weights):
    from diffusion_pipe_b200 import optim
    cfg = rec['config']
    ps = [torch.nn.Parameter(w.clone()) for w in weights]
    groups = [[p for p, (_, _, g) in zip(ps, rec['params']) if g == 0], [p for p, (_, _, g) in zip(ps, rec['params']) if g == 1]]
    extra = {k: cfg[k] for k in ('lr_bump', 'min_lr', 'max_lr', 'beta2') if k in cfg}
    opt = optim.Automagic([{'params': groups[0]}, {'params': groups[1], 'weight_decay': 0.0}], lr=cfg['lr'],
                          weight_decay=cfg['weight_decay'], clip_threshold=cfg['clip_threshold'], **extra)
    return opt, ps


def _our_state_as_reference(st):
    out = {k: v for k, v in st.items() if k not in ('lr_mask_q', 'lr_mask_scale')}
    out['lr_mask'] = {'quantized': st['lr_mask_q'], 'scale': float(st['lr_mask_scale']), 'orig_dtype': torch.float32}
    return out


def test_the_optimizer_reproduces_the_fixture_from_scratch(golden, one_thread, oracle_ops):
    """four steps of optim.Automagic (oracle-backed) from the initial weights equal the reference's four steps; the
    statistics are stored as fp32 (holding the bf16 values at step 1)"""
    for case, rec in golden['cases'].items():
        opt, ps = _fixture_optimizer(rec, rec['init'])
        for s in range(golden['steps']):
            for p, g in zip(ps, rec['grads'][s]):
                p.grad = g.clone() if g is not None else None
            opt.step()
            for i, p in enumerate(ps):
                assert torch.equal(_bits(p.detach()), _bits(rec['weights'][s][i])), (case, s, i)
                want = rec['states'][s][i]
                if want is None:
                    assert not opt.state[p]
                    continue
                mine = _our_state_as_reference(opt.state[p])
                for k, v in want.items():
                    if torch.is_tensor(v) and v.is_floating_point():
                        assert torch.equal(mine[k].to(v.dtype), v), (case, s, i, k)
                    elif k == 'lr_mask':
                        assert torch.equal(mine[k]['quantized'], v['quantized']) and mine[k]['scale'] == v['scale']
                    else:
                        assert (torch.equal(mine[k], v) if torch.is_tensor(v) else mine[k] == v), k


def test_loading_the_reference_state_dict_continues_with_the_reference_steps(golden, one_thread, oracle_ops):
    for case, rec in golden['cases'].items():
        opt, ps = _fixture_optimizer(rec, rec['weights'][1])
        opt.load_state_dict(rec['state_dict_step2'])
        steps = [opt.state[p]['step'] if opt.state[p] else 0 for p in ps]
        assert steps == [s['step'] if s is not None else 0 for s in rec['states'][1]]
        for s in (2, 3):
            for p, g in zip(ps, rec['grads'][s]):
                p.grad = g.clone() if g is not None else None
            opt.step()
            for i, p in enumerate(ps):
                assert torch.equal(_bits(p.detach()), _bits(rec['weights'][s][i])), (case, s, i)
                want = rec['states'][s][i]
                mine = _our_state_as_reference(opt.state[p])
                assert torch.equal(mine['lr_mask']['quantized'], want['lr_mask']['quantized'])
                assert mine['lr_mask']['scale'] == want['lr_mask']['scale']
                assert torch.equal(mine['avg_lr'], want['avg_lr']) and mine['step'] == want['step']


def test_state_dict_format_and_round_trip(golden, oracle_ops):
    rec = golden['cases']['bf16_mixed']
    opt, ps = _fixture_optimizer(rec, rec['init'])
    for s in range(2):
        for p, g in zip(ps, rec['grads'][s]):
            p.grad = g.clone() if g is not None else None
        opt.step()
    sd = opt.state_dict()
    for st in sd['state'].values():
        assert set(st['lr_mask']) == {'quantized', 'scale', 'orig_dtype'}
        assert st['lr_mask']['quantized'].dtype == torch.int8 and isinstance(st['lr_mask']['scale'], float)
        assert st['lr_mask']['orig_dtype'] == torch.float32
        assert 'RMS' not in st and 'lr_mask_q' not in st
        assert set(st) >= {'step', 'avg_lr', 'last_polarity', 'shift'}
    opt2, ps2 = _fixture_optimizer(rec, [p.detach() for p in ps])
    opt2.load_state_dict(sd)
    for p, q in zip(ps, ps2):
        a, b = opt.state[p], opt2.state[q]
        assert set(a) == set(b)
        for k in a:
            assert (torch.equal(a[k], b[k]) and a[k].dtype == b[k].dtype) if torch.is_tensor(a[k]) else a[k] == b[k], k
    for p, q, g in zip(ps, ps2, rec['grads'][2]):
        p.grad = q.grad = g.clone() if g is not None else None
    opt.step()
    opt2.step()
    assert all(torch.equal(_bits(p.detach()), _bits(q.detach())) for p, q in zip(ps, ps2))


def test_loading_a_state_dict_without_lr_mask_does_nothing(golden, oracle_ops):
    rec = golden['cases']['fp32_mixed']
    opt, ps = _fixture_optimizer(rec, rec['init'])
    for p, g in zip(ps, rec['grads'][0]):
        p.grad = g.clone() if g is not None else None
    opt.step()
    before = {id(p): {k: (v.clone() if torch.is_tensor(v) else v) for k, v in opt.state[p].items()} for p in ps}
    groups = [dict(g) for g in opt.param_groups]
    other = torch.optim.AdamW([torch.nn.Parameter(torch.zeros(3))], lr=0.5)
    opt.load_state_dict(other.state_dict())
    opt.load_state_dict({'state': {0: {'step': 7, 'exp_avg': torch.zeros(3)}}, 'param_groups': [{'lr': 9.0, 'params': [0]}]})
    for p in ps:
        for k, v in before[id(p)].items():
            assert (torch.equal(opt.state[p][k], v) if torch.is_tensor(v) else opt.state[p][k] == v), k
    assert [g['lr'] for g in opt.param_groups] == [g['lr'] for g in groups]


# ---------------------------------------------------------------------------------------------------------------------
# factory and constructor rules
# ---------------------------------------------------------------------------------------------------------------------
class _Model:
    def get_param_groups(self, params):
        return [{'params': params}]


@pytest.mark.parametrize('typ', ['automagic', 'Automagic'])
def test_factory_builds_automagic_with_the_wd_split(typ, capsys):
    import train as T
    from diffusion_pipe_b200 import optim
    ps = [torch.nn.Parameter(torch.zeros(4, 6, dtype=BF16)), torch.nn.Parameter(torch.zeros(6, dtype=BF16))]
    opt = T.make_optimizer_factory({'optimizer': {'type': typ, 'lr': 5e-3, 'weight_decay': 0.01, 'lr_bump': 2e-6,
                                                  'min_lr': 1e-8, 'max_lr': 1e-2, 'beta2': 0.99}}, _Model())(ps)
    assert isinstance(opt, optim.Automagic)
    assert 'Start lr is very high' in capsys.readouterr().out
    assert opt.lr == 1e-6                                             # the mask starts at 1e-6 ...
    assert [g['lr'] for g in opt.param_groups] == [5e-3, 5e-3]         # ... while group['lr'] keeps the given value
    assert [g['weight_decay'] for g in opt.param_groups] == [0.01, 0]
    assert [g['beta2'] for g in opt.param_groups] == [0.99, 0.99]
    assert (opt.lr_bump, opt.min_lr, opt.max_lr) == (2e-6, 1e-8, 1e-2)  # optimizer-wide, not per group
    assert all('lr_bump' not in g for g in opt.param_groups)
    assert opt.get_learning_rates() == [0.0, 0.0]                       # parameters without state count as 0, as in the reference


def test_constructor_defaults_and_start_mask():
    from diffusion_pipe_b200 import optim
    p = torch.nn.Parameter(torch.zeros(3, 5))
    opt = optim.Automagic([p])
    g = opt.param_groups[0]
    assert (g['lr'], g['eps'], g['clip_threshold'], g['beta2'], g['weight_decay']) == (1e-6, (1e-30, 1e-3), 1.0, 0.999, 0.0)
    st = opt._init_state(p)
    want = A.init_state(p.detach(), 1e-6)
    assert torch.equal(st['lr_mask_q'], want['lr_mask']['quantized'])
    assert float(st['lr_mask_scale']) == want['lr_mask']['scale']
    assert st['exp_avg_sq_row'].shape == (3,) and st['exp_avg_sq_col'].shape == (5,) and 'shift' not in st
    assert opt.get_learning_rates() == [float(st['avg_lr'])]


def test_parameter_swapping_and_unsupported_parameters_are_refused():
    from diffusion_pipe_b200 import optim
    p = torch.nn.Parameter(torch.zeros(4, 4, dtype=BF16))
    with pytest.raises(NotImplementedError):
        optim.Automagic([p], do_paramiter_swapping=True)
    for dt in (torch.float16, torch.float8_e4m3fn):
        with pytest.raises(TypeError):
            optim.Automagic([torch.nn.Parameter(torch.zeros(4, 4).to(dt), requires_grad=False)])
    opt = optim.Automagic([p])
    p.grad = torch.ones(4, 4, dtype=BF16)
    with pytest.raises(TypeError, match='CUDA'):                       # the step kernels refuse CPU tensors
        opt.step()


def test_other_types_still_raise():
    import train as T
    ps = [torch.nn.Parameter(torch.zeros(4, 4))]
    for typ in ('adamw8bitkahan', 'stableadamw'):
        with pytest.raises(NotImplementedError):
            T.make_optimizer_factory({'optimizer': {'type': typ, 'lr': 1e-4}}, _Model())(ps)


# ---------------------------------------------------------------------------------------------------------------------
# C ABI
# ---------------------------------------------------------------------------------------------------------------------
def test_abi_structs_match_the_c_compiler(tmp_path):
    from diffusion_pipe_b200 import _abi
    src = '#include <stdio.h>\n#include <stddef.h>\n#include "dpipe.h"\nint main(void){\n'
    for name, cls in (('dpipe_automagic_tensor', _abi.AutomagicTensor), ('dpipe_automagic_scalars', _abi.AutomagicScalars)):
        for f, _ in cls._fields_:
            src += f'  printf("{name} {f} %zu\\n", offsetof({name}, {f}));\n'
        src += f'  printf("{name} __size__ %zu\\n", sizeof({name}));\n'
    src += '  return 0; }\n'
    (tmp_path / 'off.c').write_text(src)
    subprocess.run(['gcc', '-std=c99', '-I', os.path.join(ROOT, 'include'), str(tmp_path / 'off.c'), '-o',
                    str(tmp_path / 'off')], check=True)
    out = subprocess.run([str(tmp_path / 'off')], check=True, capture_output=True, text=True).stdout.split()
    got = {(out[i], out[i + 1]): int(out[i + 2]) for i in range(0, len(out), 3)}
    for name, cls in (('dpipe_automagic_tensor', _abi.AutomagicTensor), ('dpipe_automagic_scalars', _abi.AutomagicScalars)):
        for f, _ in cls._fields_:
            assert getattr(cls, f).offset == got[(name, f)], (name, f)
        assert ctypes.sizeof(cls) == got[(name, '__size__')]


def _lib_or_skip():
    from diffusion_pipe_b200 import _lib
    try:
        return _lib.lib()
    except Exception as e:                                            # noqa: BLE001
        pytest.skip(f'native library not loadable here: {e}')


def test_entry_points_reject_bad_arguments_before_any_cuda_call():
    from diffusion_pipe_b200 import _abi
    lib = _lib_or_skip()
    t = (_abi.AutomagicTensor * 1)()
    sc = _abi.AutomagicScalars(0.999, 1e-30, 1e-6, 1e-7, 1e-3, 1.0, 0.0)
    dummy = ctypes.c_void_p(16)
    for f in ('p', 'g', 'row', 'col', 'v', 'code', 'pol', 'shift', 'scale', 'avg_lr', 'ws'):
        setattr(t[0], f, dummy)
    t[0].numel, t[0].L, t[0].R, t[0].C, t[0].dtype, t[0].flags = 12, 1, 3, 4, 0, 1

    def rc(**fields):
        a = (_abi.AutomagicTensor * 1)()
        ctypes.memmove(a, t, ctypes.sizeof(t))
        for k, v in fields.items():
            setattr(a[0], k, v)
        return (lib.dpipe_automagic_apply(a, 1, ctypes.byref(sc), None),
                lib.dpipe_automagic_stats(a, 1, ctypes.byref(sc), None, 0, None))
    for bad in (dict(dtype=2), dict(C=5), dict(flags=8), dict(shift=None), dict(dtype=1, flags=3), dict(row=None),
                dict(flags=0, v=None), dict(numel=-1), dict(code=None)):
        assert all(r < 0 for r in rc(**bad)), bad
    assert lib.dpipe_automagic_apply(t, -1, ctypes.byref(sc), None) < 0
    assert lib.dpipe_automagic_apply(t, 1, None, None) < 0
    bad_clip = _abi.AutomagicScalars(0.999, 1e-30, 1e-6, 1e-7, 1e-3, 0.0, 0.0)
    assert lib.dpipe_automagic_apply(t, 1, ctypes.byref(bad_clip), None) < 0
