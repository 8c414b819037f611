"""CPU: the CAME optimizer (`type = 'CAME'`) — the kernels' specification (oracle/came_ref.py emulation) against the
recalled torch-op text, factored and 1-D paths, steps with and without clipping, tracking fp64 CAME on a convex
quadratic, the optimizer factory and constructor rules, the state dict and resume (with `ops.came_*` replaced by an
emulation-backed double defined in this file), a CLI run on the kernel doubles, and the C entry points' argument
checks."""
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

from oracle import came_ref as CR  # noqa: E402

BF16 = torch.bfloat16
SHAPES = [(7,), (64, 33), (3, 5, 7), (1000,), (17, 241), (), (2, 3, 4, 5)]
STATE_KEYS = ('exp_avg', 'exp_avg_sq', 'exp_avg_sq_row', 'exp_avg_sq_col', 'exp_avg_res_row', 'exp_avg_res_col')


def _bits(t):
    return t.view(torch.int16) if t.dtype == BF16 else t.view(torch.int32) if t.dtype == torch.float32 else t


def _groups(dtype, seed=0, lr=1e-3):
    gen = torch.Generator().manual_seed(seed)
    ps = [(torch.randn(s, generator=gen) * 0.05).to(dtype) for s in SHAPES]
    return [dict(CR.DEFAULTS, lr=lr, weight_decay=0.01, params=ps[:4]),
            dict(CR.DEFAULTS, lr=2 * lr, weight_decay=0.0, params=ps[4:])], gen


def _grads(groups, gen, drop=None):
    out, k = [], 0
    for g in groups:
        gl = []
        for p in g['params']:
            gl.append(None if k == drop else (torch.randn(p.shape, generator=gen) * 1e-2).to(p.dtype))
            k += 1
        out.append(gl)
    return out


def agree(a, b, dtype, ref, weights=None):
    """the tolerance between the specification and the torch-op text: the two round the same ops, but torch reduces
    in fp32 in its own order (on CUDA it also takes an approximate rsqrt; on CPU a bf16 add rounds its alpha to bf16
    first), so a row or column factor can differ by an ulp, which moves whole rows by an ulp and, through res, the
    next step's factors; the residual (u - m)^2 doubles u's relative error.  fp32: within 1e-5 of the largest
    magnitude of `ref`; bf16: within 2^-5 of it (four bf16 ulps at the largest element).  For a step change of the weights (`weights`: the weights before the step) one more ulp
    of the largest weight, the rounding of the new weight (2^-22 / 2^-7 relative)"""
    if not a.numel():
        return True
    tol = (1e-5 if dtype == torch.float32 else 2.0 ** -5) * float(ref.float().abs().max())
    if weights is not None:
        tol += (2.0 ** -22 if dtype == torch.float32 else 2.0 ** -7) * float(weights.float().abs().max())
    return float((a.float() - b.float()).abs().max()) <= tol


@pytest.mark.parametrize('dtype', [torch.float32, BF16])
@pytest.mark.parametrize('clip', [1.0, 1e4])
def test_emulation_agrees_with_the_torch_op_text(dtype, clip):
    """three steps, two groups with different lr and wd, one parameter without a gradient at step 2; with
    clip_threshold 1 every step clips (rms(u) starts near 1 / sqrt(1 - beta2)), with 1e4 none does.  The state after
    each step within `agree` of the text's; the weights' step changes within `agree` of the text's change"""
    groups, gen = _groups(dtype)
    emu = copy.deepcopy(groups)
    ts, es = {}, {}
    for step in range(3):
        grads = _grads(groups, gen, drop=1 if step == 1 else None)
        before = [p.clone() for g in groups for p in g['params']]
        ebefore = [p.clone() for g in emu for p in g['params']]
        for g, gl in zip(emu, grads):
            for p, grad in zip(g['params'], gl):
                if grad is not None:
                    st = es.get(id(p)) or CR.init_state(p)
                    _, _, _, cd = CR.came_param_emulated(p, grad, st, lr=g['lr'], betas=g['betas'],
                                                         weight_decay=g['weight_decay'], fixed_decay=False,
                                                         eps1=g['eps1'], eps2=g['eps2'], clip_threshold=clip)
                    assert (cd > 1.0) if clip == 1.0 else (cd == 1.0), (step, tuple(p.shape), cd)
        CR.came_step_torch_ops(groups, grads, ts, clip)
        CR.came_step_emulated(emu, grads, es, clip)
        tp = [p for g in groups for p in g['params']]
        ep = [p for g in emu for p in g['params']]
        for k, (a, b, e0, p0) in enumerate(zip(ep, tp, ebefore, before)):
            da, db = a.float() - e0.float(), b.float() - p0.float()
            assert agree(da, db, dtype, db, p0), (step, k, tuple(a.shape))
            if step == 1 and k == 1:
                assert torch.equal(_bits(a), _bits(e0)) and torch.equal(_bits(b), _bits(p0))
        for (pe, pt) in zip(ep, tp):
            if id(pt) not in ts:
                continue
            for key in STATE_KEYS:
                if key in ts[id(pt)]:
                    assert agree(es[id(pe)][key], ts[id(pt)][key], dtype, ts[id(pt)][key]), (step, key, tuple(pt.shape))
            assert es[id(pe)]['step'] == ts[id(pt)]['step']


def test_factored_and_one_d_paths_and_their_state():
    """ndim >= 2 keeps four row / column vectors (over the last two dims, leading dims kept); 1-D and 0-D keep a
    param-shaped exp_avg_sq; every state tensor is in the parameter's dtype"""
    for dtype in (torch.float32, BF16):
        for shape, want in (((7,), {'exp_avg_sq': (7,)}), ((), {'exp_avg_sq': ()}),
                            ((3, 5, 7), {'exp_avg_sq_row': (3, 5), 'exp_avg_sq_col': (3, 7), 'exp_avg_res_row': (3, 5),
                                         'exp_avg_res_col': (3, 7)})):
            st = CR.init_state(torch.zeros(shape, dtype=dtype))
            assert {k: tuple(v.shape) for k, v in st.items() if k not in ('step', 'exp_avg')} == want
            assert all(v.dtype == dtype for k, v in st.items() if k != 'step')


def test_specification_with_given_sums_is_the_one_without():
    """feeding the emulation its own fp64 sums changes nothing (the GPU test feeds it the kernels' sums)"""
    gen = torch.Generator().manual_seed(5)
    for shape in ((17, 241), (3, 5, 7), (9,)):
        p = torch.randn(shape, generator=gen) * 0.05
        st = CR.init_state(p)
        st['exp_avg'] = torch.randn(shape, generator=gen) * 1e-3
        g = torch.randn(shape, generator=gen) * 1e-2
        kw = dict(lr=1e-3, betas=(0.9, 0.999, 0.9999), weight_decay=0.01, fixed_decay=True, eps1=1e-30, eps2=1e-16,
                  clip_threshold=1.0)
        a, sa, own, ca = CR.came_param_emulated(p, g, st, **kw)
        b, sb, _, cb = CR.came_param_emulated(p, g, st, sums=own, **kw)
        assert torch.equal(a, b) and ca == cb and all(torch.equal(sa[k], sb[k]) for k in sa)


def test_tracks_fp64_came_on_a_convex_quadratic():
    """fp32 emulation against the text in fp64 on sum (p - target)^2 / 2: the loss falls by half and the weights stay
    within 1e-4 of the fp64 run (relative to the target's scale) over 40 steps"""
    gen = torch.Generator().manual_seed(3)
    target = torch.randn(64, 48, generator=gen)
    tb = torch.randn(48, generator=gen)
    p32, b32 = torch.zeros(64, 48), torch.zeros(48)
    p64, b64 = p32.double(), b32.double()
    g32 = [dict(CR.DEFAULTS, lr=3e-2, params=[p32, b32])]
    g64 = [dict(CR.DEFAULTS, lr=3e-2, params=[p64, b64])]
    s32, s64 = {}, {}
    loss0 = float(((p64 - target.double()) ** 2).sum() / 2)
    for _ in range(40):
        CR.came_step_emulated(g32, [[p32 - target, b32 - tb]], s32)
        CR.came_step_torch_ops(g64, [[p64 - target.double(), b64 - tb.double()]], s64)
        assert float((p32.double() - p64).abs().max()) <= 1e-4 * float(target.abs().max())
        assert float((b32.double() - b64).abs().max()) <= 1e-4 * float(tb.abs().max())
    assert float(((p64 - target.double()) ** 2).sum() / 2) < 0.5 * loss0


# ---------------------------------------------------------------------------------------------------------------------
# the optimizer on CPU, with the kernels replaced by the emulation
# ---------------------------------------------------------------------------------------------------------------------
class _Args:
    """the test double of ops.CameArgs: the packed state and options, no gradients"""
    packs = 0

    def __init__(self, params, m, row, col, res_row, res_col, v, weight_decay, betas, eps1, eps2, fixed_decay):
        type(self).packs += 1
        self.params = params
        self.state = [dict(exp_avg=m[i], exp_avg_sq_row=row[i], exp_avg_sq_col=col[i], exp_avg_res_row=res_row[i],
                           exp_avg_res_col=res_col[i], exp_avg_sq=v[i]) for i in range(len(params))]
        self.opts = list(zip(weight_decay, betas, eps1, eps2, fixed_decay))


def _emu_step(args, grads, lrs, clip_threshold):
    for p, g, lr, st, (wd, betas, e1, e2, fixed) in zip(args.params, grads, lrs, args.state, args.opts):
        if p.device.type != 'cpu' or g is None or g.shape != p.shape:
            raise TypeError('came: the test double takes CPU tensors with a gradient of the parameter shape')
        pn, new, _, _ = CR.came_param_emulated(p, g, {k: v for k, v in st.items() if v is not None}, lr=lr, betas=betas,
                                               weight_decay=wd, fixed_decay=fixed, eps1=e1, eps2=e2,
                                               clip_threshold=clip_threshold)
        for k, v in new.items():
            st[k].copy_(v)
        p.data.copy_(pn)


@pytest.fixture
def emu_ops(monkeypatch):
    from diffusion_pipe_b200 import ops
    monkeypatch.setattr(ops, 'came_pack', _Args)
    monkeypatch.setattr(ops, 'came_step', _emu_step)


def _optimizer(weights, **kw):
    from diffusion_pipe_b200 import optim
    ps = [torch.nn.Parameter(w.clone()) for w in weights]
    opt = optim.CAME([{'params': ps[:4]}, {'params': ps[4:], 'weight_decay': 0.0, 'lr': 2e-3}], lr=1e-3,
                     weight_decay=0.01, **kw)
    return opt, ps


def _step(opt, ps, gen, skip=None):
    for i, p in enumerate(ps):
        p.grad = None if i == skip else (p.detach().float() * 0.5 + torch.randn(p.shape, generator=gen) * 1e-2).to(p.dtype)
    opt.step()


def test_the_optimizer_follows_the_emulation_and_reads_lr_each_step(emu_ops):
    gen = torch.Generator().manual_seed(0)
    ws = [(torch.randn(s, generator=gen) * 0.05).to(dt) for s, dt in zip(SHAPES, (BF16, torch.float32) * 4)]
    opt, ps = _optimizer(ws)
    groups = [dict(CR.DEFAULTS, lr=1e-3, weight_decay=0.01, params=[w.clone() for w in ws[:4]]),
              dict(CR.DEFAULTS, lr=2e-3, weight_decay=0.0, params=[w.clone() for w in ws[4:]])]
    states = {}
    g1, g2 = torch.Generator().manual_seed(1), torch.Generator().manual_seed(1)
    for s in range(4):
        if s == 2:                      # an LR scheduler's change reaches the next step
            opt.param_groups[0]['lr'] = groups[0]['lr'] = 5e-4
        _step(opt, ps, g1, skip=3 if s == 1 else None)
        grads = [[None if (s == 1 and gi == 0 and k == 3) else
                  (p.float() * 0.5 + torch.randn(p.shape, generator=g2) * 1e-2).to(p.dtype)
                  for k, p in enumerate(g['params'])] for gi, g in enumerate(groups)]
        CR.came_step_emulated(groups, grads, states)
        want = [p for g in groups for p in g['params']]
        assert all(torch.equal(_bits(a.detach()), _bits(b)) for a, b in zip(ps, want)), s
    assert opt.state[ps[3]]['step'] == 3 and opt.state[ps[0]]['step'] == 4


def test_gradients_are_not_kept_and_the_pack_is_reused(emu_ops):
    import gc
    import weakref
    gen = torch.Generator().manual_seed(4)
    ws = [(torch.randn(s, generator=gen) * 0.05).to(BF16) for s in SHAPES]
    opt, ps = _optimizer(ws)
    _Args.packs = 0
    for k in range(3):
        opt.param_groups[1]['lr'] = 1e-3 * (k + 1)           # lr changes do not repack
        _step(opt, ps, gen)
        refs = [weakref.ref(p.grad) for p in ps]
        opt.zero_grad(set_to_none=True)
        gc.collect()
        assert all(r() is None for r in refs)
    assert _Args.packs == 1
    _step(opt, ps, gen, skip=2)                               # another set of parameters with gradients: packed anew
    assert _Args.packs == 2


def test_state_dict_round_trip_resume_and_the_reference_layout(emu_ops):
    gen = torch.Generator().manual_seed(2)
    ws = [(torch.randn(s, generator=gen) * 0.05).to(BF16) for s in SHAPES]
    opt, ps = _optimizer(ws)
    g = torch.Generator().manual_seed(7)
    for _ in range(3):
        _step(opt, ps, g)
    sd = opt.state_dict()
    assert set(sd['state'][1]) == {'step', 'exp_avg', 'exp_avg_sq_row', 'exp_avg_sq_col', 'exp_avg_res_row',
                                   'exp_avg_res_col'}
    assert set(sd['state'][0]) == {'step', 'exp_avg', 'exp_avg_sq'} and sd['state'][0]['step'] == 3
    opt2, ps2 = _optimizer([p.detach() for p in ps])
    opt2.load_state_dict(copy.deepcopy(sd))
    ref = copy.deepcopy(sd)                                  # pytorch_optimizer's layout: an `RMS` entry per parameter
    for st in ref['state'].values():
        st['RMS'] = torch.tensor(0.05)
    opt3, ps3 = _optimizer([p.detach() for p in ps])
    opt3.load_state_dict(ref)
    assert all('RMS' not in st for st in opt3.state.values())
    gens = [torch.Generator().manual_seed(9) for _ in range(3)]
    for _ in range(2):
        for o, q, gg in ((opt, ps, gens[0]), (opt2, ps2, gens[1]), (opt3, ps3, gens[2])):
            _step(o, q, gg)
    for q in (ps2, ps3):
        assert all(torch.equal(_bits(a.detach()), _bits(b.detach())) for a, b in zip(ps, q))


# ---------------------------------------------------------------------------------------------------------------------
# factory and constructor rules
# ---------------------------------------------------------------------------------------------------------------------
class _Model:
    def get_param_groups(self, params):
        return [{'params': params}]


@pytest.mark.parametrize('typ', ['CAME', 'came'])
def test_factory_builds_came_with_the_wd_split(typ):
    import train as T
    from diffusion_pipe_b200 import optim
    ps = [torch.nn.Parameter(torch.zeros(4, 6, dtype=BF16)), torch.nn.Parameter(torch.zeros(6, dtype=BF16))]
    opt = T.make_optimizer_factory({'optimizer': {'type': typ, 'lr': 1e-4, 'weight_decay': 0.01}}, _Model())(ps)
    assert isinstance(opt, optim.CAME)
    g0, g1 = opt.param_groups
    for k, v in CR.DEFAULTS.items():
        if k not in ('lr', 'weight_decay'):
            assert g0[k] == v and g1[k] == v, k
    assert (g0['lr'], g0['weight_decay'], g1['weight_decay']) == (1e-4, 0.01, 0)
    assert g0['params'][0] is ps[0] and g1['params'][0] is ps[1]
    assert opt.clip_threshold == 1.0
    opt = T.make_optimizer_factory({'optimizer': {'type': typ, 'betas': [0.9, 0.99, 0.999], 'clip_threshold': 2.0,
                                                  'eps1': 1e-20}}, _Model())(ps)
    assert opt.param_groups[0]['betas'] == (0.9, 0.99, 0.999) and opt.clip_threshold == 2.0
    assert opt.param_groups[0]['eps1'] == 1e-20


def test_refused_options_and_unknown_kwargs():
    import train as T
    from diffusion_pipe_b200 import optim
    p = torch.nn.Parameter(torch.zeros(4, 4, dtype=BF16))
    with pytest.raises(TypeError):
        optim.CAME([p], not_an_option=1)
    for kw in (dict(ams_bound=True), dict(maximize=True), dict(weight_decouple=False), dict(gradient_release=True)):
        with pytest.raises(NotImplementedError):
            optim.CAME([p], **kw)
    with pytest.raises(NotImplementedError):
        T.make_optimizer_factory({'optimizer': {'type': 'CAME', 'gradient_release': True}}, _Model())([p])
    for kw in (dict(betas=(0.9, 0.999)), dict(betas=(0.9, 1.0, 0.9)), dict(lr=-1.0), dict(clip_threshold=0.0)):
        with pytest.raises(ValueError):
            optim.CAME([p], **kw)
    for dt in (torch.float16, torch.float8_e4m3fn):
        with pytest.raises(TypeError):
            optim.CAME([torch.nn.Parameter(torch.zeros(4, 4).to(dt), requires_grad=False)])
    opt = optim.CAME([p])
    p.grad = torch.ones(4, 4, dtype=BF16)
    with pytest.raises(TypeError, match='CUDA'):
        opt.step()
    for typ in ('adamw8bitkahan', 'stableadamw', 'lion'):
        with pytest.raises(NotImplementedError):
            T.make_optimizer_factory({'optimizer': {'type': typ, 'lr': 1e-4}}, _Model())([p])


def test_cli_run_with_the_emulated_ops_and_resume(tmp_path, monkeypatch, emu_ops):
    """train.py on a small Flux model with the kernel doubles and `type = 'CAME'`: the loss is logged every step and
    a run resumed from the step-2 checkpoint logs the same step-3 loss"""
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
checkpoint_every_n_steps = 2
max_steps = 3
eval_before_first_step = false
[model]
type = 'flux'
dtype = 'bfloat16'
device = 'cpu'
transformer_config = {{ num_attention_heads = 2, num_layers = 1, num_single_layers = 1, joint_attention_dim = 64, pooled_projection_dim = 32 }}
[optimizer]
type = 'CAME'
lr = 1e-4
weight_decay = 0.01
""")
    run_dir = T.main(['--config', str(cfgp)])
    lines = [json.loads(line) for line in open(os.path.join(run_dir, 'metrics.jsonl'))]
    losses = [line for line in lines if line['tag'] == 'train/loss']
    assert [line['x'] for line in losses] == [1, 2, 3]
    assert all(line['value'] == line['value'] for line in losses)          # finite, not NaN


# ---------------------------------------------------------------------------------------------------------------------
# C ABI
# ---------------------------------------------------------------------------------------------------------------------
def test_abi_struct_matches_the_c_compiler(tmp_path):
    from diffusion_pipe_b200 import _abi
    name, cls = 'dpipe_came_tensor', _abi.CameTensor
    src = '#include <stdio.h>\n#include <stddef.h>\n#include "dpipe.h"\nint main(void){\n'
    for f, _ in cls._fields_:
        src += f'  printf("{f} %zu\\n", offsetof({name}, {f}));\n'
    src += f'  printf("__size__ %zu\\n", sizeof({name}));\n  return 0; }}\n'
    (tmp_path / 'off.c').write_text(src)
    subprocess.run(['gcc', '-std=c99', '-I', os.path.join(ROOT, 'include'), str(tmp_path / 'off.c'), '-o',
                    str(tmp_path / 'off')], check=True)
    out = subprocess.run([str(tmp_path / 'off')], check=True, capture_output=True, text=True).stdout.split()
    got = {out[i]: int(out[i + 1]) for i in range(0, len(out), 2)}
    for f, _ in cls._fields_:
        assert getattr(cls, f).offset == got[f], f
    assert ctypes.sizeof(cls) == got['__size__']


def _lib_or_skip():
    from diffusion_pipe_b200 import _lib
    try:
        return _lib.lib()
    except Exception as e:                                            # noqa: BLE001
        pytest.skip(f'native library not loadable here: {e}')


def test_entry_points_reject_bad_arguments_before_any_cuda_call():
    """fake pointers throughout: every call below must fail in the host checks (a launch would fault)"""
    from diffusion_pipe_b200 import _abi
    lib = _lib_or_skip()
    t = (_abi.CameTensor * 1)()
    for f in ('p', 'g', 'm', 'row', 'col', 'res_row', 'res_col', 'fac', 'sums'):
        setattr(t[0], f, ctypes.c_void_p(64))
    t[0].numel, t[0].L, t[0].R, t[0].C, t[0].dtype, t[0].factored = 12, 1, 3, 4, 0, 1
    t[0].lr, t[0].beta1, t[0].beta2, t[0].beta3, t[0].eps1, t[0].eps2 = 1e-3, 0.9, 0.999, 0.9999, 1e-30, 1e-16
    scratch = ctypes.c_void_p(128)
    need = ctypes.c_int64()
    assert lib.dpipe_came_scratch_doubles(t, 1, ctypes.byref(need)) == 0
    assert need.value == 3 + 4 + 1        # one row strip of 3 partials, one row block of 4 column partials, one CTA

    def rc(a, n=1, clip=1.0, scr=scratch, length=1 << 20):
        return lib.dpipe_came_step(a, n, clip, scr, length, None)
    for bad in (dict(dtype=2), dict(numel=-1), dict(g=None), dict(m=None), dict(res_col=None), dict(fac=None),
                dict(sums=None), dict(C=5), dict(L=0), dict(p=ctypes.c_void_p(65)), dict(beta3=1.0), dict(beta1=-0.1),
                dict(eps2=-1.0), dict(lr=float('nan')), dict(weight_decay=-1.0), dict(factored=0)):
        a = (_abi.CameTensor * 1)()
        ctypes.memmove(a, t, ctypes.sizeof(t))
        for k, v in bad.items():
            setattr(a[0], k, v)
        assert rc(a) < 0, bad
        assert b'dpipe_came_step' in lib.dpipe_last_error(), bad
    assert rc(t, n=-1) < 0
    assert rc(t, clip=0.0) < 0 and b'clip_threshold' in lib.dpipe_last_error()
    assert rc(t, length=7) < 0 and b'scratch' in lib.dpipe_last_error()
    assert rc(t, scr=None) < 0
    assert lib.dpipe_came_scratch_doubles(t, 1, None) < 0
