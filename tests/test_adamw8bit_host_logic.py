"""CPU: the AdamW8bit optimizer (`type = 'adamw8bit'`) — bnb's dynamic maps and the nearest-entry quantizer, the
kernel's specification (oracle/adamw8bit_ref.py) against an fp64 restatement (32-bit path) and against fp64 AdamW on a
convex quadratic (8-bit path), the all-zero-gradient block of a LoRA factor at step 1, non-finite gradients, the
optimizer factory and constructor rules, the state dict and resume and a CLI run (with `ops.adamw8bit_step` replaced by
an emulation-backed double defined in this file), and the C entry point's argument checks."""
import copy
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (ROOT, HERE):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from oracle import adamw8bit_ref as A  # noqa: E402

BF16 = torch.bfloat16


def _bits(t):
    return t.view(torch.int16) if t.dtype == BF16 else t.view(torch.int32) if t.dtype == torch.float32 else t


def test_maps_are_bnbs_dynamic_maps():
    from diffusion_pipe_b200 import optim
    for signed in (True, False):
        q = A.create_dynamic_map(signed)
        assert q.shape == (256,) and q.dtype == torch.float32
        assert bool((q[1:] > q[:-1]).all())
        assert 0.0 in q.tolist() and 1.0 in q.tolist() and float(q[-1]) == 1.0
        assert torch.equal(optim.dynamic_map(signed), q)                  # the package's copy of the construction
    q = A.create_dynamic_map(True)
    neg, zero, pos = q[:127], q[127], q[128:255]
    assert float(zero) == 0.0 and torch.equal(-neg.flip(0), pos)            # mirrored, apart from 1.0
    u = A.create_dynamic_map(False)
    assert float(u[0]) == 0.0 and float(u[1]) > 0


@pytest.mark.parametrize('signed', [True, False])
def test_quantizer_returns_a_nearest_entry(signed):
    """on a dense sweep of [-1, 1] (or [0, 1]) plus every midpoint and its fp32 neighbours: the entry is nearest, up to
    the fp32 rounding of the midpoint that decides between two neighbours; exactly at a midpoint it is the lower one"""
    q = A.create_dynamic_map(signed).numpy()
    mid = A.midpoints(q)
    lo = -1.0 if signed else 0.0
    sweep = np.concatenate([np.linspace(lo, 1.0, 200001, dtype=np.float32), mid, np.nextafter(mid, np.float32(2)),
                            np.nextafter(mid, np.float32(-2)), q, np.float32([0.0, -0.0, 1e-30, -1e-30])])
    if not signed:
        sweep = sweep[sweep >= 0]
    c = A.quantize(q, sweep).astype(np.int64)
    d = np.abs(sweep.astype(np.float64) - q[c].astype(np.float64))
    best = np.abs(sweep.astype(np.float64)[:, None] - q.astype(np.float64)[None, :]).min(axis=1)
    slack = np.abs(mid.astype(np.float64)).max() * 2.0 ** -23
    assert bool((d <= best + slack).all())
    assert bool((d[np.abs(d - best) > 0] <= best[np.abs(d - best) > 0] + 2.0 ** -24).all())
    assert (A.quantize(q, mid).astype(np.int64) == np.arange(255)).all()            # ties go down
    assert (A.quantize(q, q).astype(np.int64) == np.arange(256)).all()              # every entry maps to itself
    assert int(A.quantize(q, np.float32([np.nan]))[0]) == 0


def _f64_32bit(p, g, m, v, sc):
    """the 32-bit path in fp64, rounded to fp32 after every operation (and to the parameter dtype where specified)"""
    def r(x):
        return torch.as_tensor(x, dtype=torch.float64).float().double()
    b1, b2 = sc['beta1'], sc['beta2']
    m = r(r(m.double() * b1) + r(r(1.0 - b1) * g.double()))
    v = r(r(v.double() * b2) + r(r(r(1.0 - b2) * g.double()) * g.double()))
    upd = r(sc['step_size'] * r(m / r(r(v.sqrt()) + sc['eps_c2'])))
    pn = r(p.double() + upd).to(p.dtype).double()
    pn = r(pn * sc['decay']).to(p.dtype)
    return pn, m.float(), v.float()


@pytest.mark.parametrize('dtype', [torch.float32, BF16])
def test_32bit_path_equals_an_fp64_restatement(dtype):
    gen = torch.Generator().manual_seed(0)
    for shape in ((7,), (64, 33), (4095,), ()):
        p = (torch.randn(shape, generator=gen) * 0.05).to(dtype)
        m = torch.randn(shape, generator=gen) * 1e-3
        v = torch.rand(shape, generator=gen) * 1e-6
        for t in (1, 2, 50):
            g = (torch.randn(shape, generator=gen) * 1e-2).to(dtype)
            sc = A.step_scalars(1e-3, (0.9, 0.999), 1e-8, 0.01, t)
            pn, m2, v2, a1, a2 = A.adamw8bit_emulated(p, g, m, v, **sc)
            wp, wm, wv = _f64_32bit(p, g, m, v, sc)
            assert a1 is None and a2 is None
            assert torch.equal(_bits(pn), _bits(wp)) and torch.equal(_bits(m2), _bits(wm)) and torch.equal(_bits(v2), _bits(wv))
            p, m, v = pn, m2, v2


def test_optimizer_scalars_are_the_specifications():
    from diffusion_pipe_b200 import optim
    for args in ((1e-3, (0.9, 0.999), 1e-8, 1e-2, 1), (3e-5, (0.95, 0.99), 1e-6, 0.0, 17), (1.0, (0.0, 0.5), 0.0, 0.1, 3)):
        assert optim.adamw8bit_scalars(*args) == A.step_scalars(*args)


def _adamw_f64(p0, target, steps, lr, betas, eps, wd):
    """AdamW with bnb's placement of eps and weight decay, in fp64"""
    p = p0.double().clone()
    m = torch.zeros_like(p)
    v = torch.zeros_like(p)
    b1, b2 = betas
    out = []
    for t in range(1, steps + 1):
        g = p - target
        m = m * b1 + (1 - b1) * g
        v = v * b2 + (1 - b2) * g * g
        c2 = (1 - b2 ** t) ** 0.5
        p = p - lr * c2 / (1 - b1 ** t) * m / (v.sqrt() + eps * c2)
        p = p * (1 - lr * wd)
        out.append(p.clone())
    return out


def test_8bit_path_tracks_fp64_adamw_on_a_convex_quadratic():
    """gradient p - target on 8192 fp32 elements (blocks of scales 1e-3 to 1), 300 steps: every 50 steps the 8-bit
    trajectory stays within 5 % of the distance fp64 AdamW has travelled (3.7 % at step 50, from the quantized early
    moments), within 1 % from step 150 on, and ends with a loss within 5 % of fp64's"""
    gen = torch.Generator().manual_seed(5)
    n = 8192
    target = torch.randn(n, generator=gen) * torch.logspace(-3, 0, n // 256).repeat_interleave(256)
    p0 = torch.zeros(n)
    hp = dict(lr=1e-2, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2)
    ref = _adamw_f64(p0, target.double(), 300, hp['lr'], hp['betas'], hp['eps'], hp['weight_decay'])
    p, st = p0.clone(), A.init_state(p0)
    assert st['state1'].dtype == torch.uint8
    for t in range(300):
        p = A.step_emulated(p, p - target, st, **hp)
        if (t + 1) % 50 == 0:
            err = float((p.double() - ref[t]).norm() / (ref[t] - p0.double()).norm())
            assert err <= (0.05 if t + 1 < 150 else 0.01), (t + 1, err)
    loss0 = float(((p0 - target) ** 2).sum())
    assert float(((p - target) ** 2).sum()) <= 1.05 * float(((ref[-1] - target.double()) ** 2).sum()) + 1e-6 * loss0


def test_zero_gradient_block_at_step_one_stays_finite():
    """a LoRA `A` factor at step 1 (B starts at zero, so A's gradient is zero): absmax 0, codes that dequantize to 0,
    p only decayed; its next, non-zero gradient starts the moments as from zero"""
    for dtype in (torch.float32, BF16):
        gen = torch.Generator().manual_seed(1)
        p = (torch.randn(32, 4096, generator=gen) * 0.02).to(dtype)
        st = A.init_state(p)
        p1 = A.step_emulated(p, torch.zeros_like(p), st)
        assert bool(torch.isfinite(p1.float()).all())
        assert not st['absmax1'].any() and not st['absmax2'].any()
        sc = A.step_scalars(1e-3, (0.9, 0.999), 1e-8, 1e-2, 1)
        want = (p.float() * sc['decay']).to(dtype)
        assert torch.equal(_bits(p1), _bits(want))
        g = (torch.randn(p.shape, generator=gen) * 1e-3).to(dtype)
        fresh = A.init_state(p)
        fresh['step'] = 1
        p2 = A.step_emulated(p1, g, st)
        p2f = A.step_emulated(p1, g, fresh)
        assert torch.equal(_bits(p2), _bits(p2f)) and bool(torch.isfinite(p2.float()).all())
        assert torch.equal(st['state1'], fresh['state1']) and torch.equal(st['absmax1'], fresh['absmax1'])


def test_non_finite_gradients():
    """8-bit path: an element whose gradient is inf or NaN keeps its p and gets m = v = 0; the rest of its block steps
    as if that element's moments were zero.  32-bit path (no skip, as bnb's 32-bit kernel): NaN reaches p"""
    gen = torch.Generator().manual_seed(2)
    p = (torch.randn(4096, generator=gen) * 0.02).to(BF16)
    st = A.init_state(p)
    p = A.step_emulated(p, (torch.randn(4096, generator=gen) * 1e-3).to(BF16), st)
    g = (torch.randn(4096, generator=gen) * 1e-3).to(BF16)
    bad = [3, 300, 301, 4095]
    g[3], g[300], g[301], g[4095] = float('inf'), float('nan'), float('-inf'), float('nan')
    sc = A.step_scalars(1e-3, (0.9, 0.999), 1e-8, 1e-2, 2)
    pn, s1, s2, a1, a2 = A.adamw8bit_emulated(p, g, st['state1'], st['state2'], st['absmax1'], st['absmax2'],
                                              st['qmap1'], st['qmap2'], **sc)
    assert torch.equal(_bits(pn[bad]), _bits(p[bad]))
    q1, q2 = st['qmap1'], st['qmap2']
    assert all(float(q1[int(s1[i])] * a1[i // 256]) == 0.0 and float(q2[int(s2[i])] * a2[i // 256]) == 0.0 for i in bad)
    assert bool(torch.isfinite(pn.float()).all()) and bool(torch.isfinite(a1).all()) and bool(torch.isfinite(a2).all())
    ok = torch.ones(4096, dtype=torch.bool)
    ok[bad] = False
    assert not torch.equal(_bits(pn[ok]), _bits(p[ok]))
    small = torch.zeros(10)
    gsm = torch.full((10,), 1e-3)
    gsm[4] = float('nan')
    pn, m, v, _, _ = A.adamw8bit_emulated(small, gsm, torch.zeros(10), torch.zeros(10), **sc)
    assert bool(torch.isnan(pn[4])) and bool(torch.isnan(m[4])) and int(torch.isnan(pn).sum()) == 1


def test_first_moment_keeps_its_sign():
    """a negative m too small for the smallest negative entry maps to it rather than to 0 (bnb's sign rule); a positive
    one rounds to 0"""
    p = torch.zeros(4096)
    st = A.init_state(p)
    g = torch.full((4096,), 1.0)
    g[7], g[8] = -1e-9, 1e-9                         # |m| / absmax = 1e-9: below half the smallest entry (5.5e-7)
    A.step_emulated(p, g, st)
    q1 = st['qmap1']
    assert float(q1[int(st['state1'][7])]) < 0 and float(q1[int(st['state1'][8])]) == 0.0


# ---------------------------------------------------------------------------------------------------------------------
# the optimizer on CPU, with the kernel replaced by the emulation
# ---------------------------------------------------------------------------------------------------------------------
def _emu_step(params, grads, state1, state2, absmax1, absmax2, scalars, qmap1=None, qmap2=None):
    for i, p in enumerate(params):
        q8 = absmax1[i] is not None
        pn, s1, s2, a1, a2 = A.adamw8bit_emulated(p.detach(), grads[i], state1[i], state2[i], absmax1[i], absmax2[i],
                                                  qmap1 if q8 else None, qmap2 if q8 else None, **scalars[i])
        p.data.copy_(pn)
        state1[i].copy_(s1)
        state2[i].copy_(s2)
        if q8:
            absmax1[i].copy_(a1)
            absmax2[i].copy_(a2)


@pytest.fixture
def emu_ops(monkeypatch):
    from diffusion_pipe_b200 import ops
    monkeypatch.setattr(ops, 'adamw8bit_step', _emu_step)


SHAPES = [(64, 96), (96,), (40, 130), (5000,), (3, 5), (257, 16)]


def _optimizer(weights, **kw):
    from diffusion_pipe_b200 import optim
    ps = [torch.nn.Parameter(w.clone()) for w in weights]
    opt = optim.AdamW8bit([{'params': ps[:4]}, {'params': ps[4:], 'weight_decay': 0.0, 'lr': 2e-3}], **kw)
    return opt, ps


def _weights(seed):
    gen = torch.Generator().manual_seed(seed)
    return [(torch.randn(s, generator=gen) * 0.05).to(dt) for s, dt in zip(SHAPES, (BF16, torch.float32) * 3)]


def _step(opt, ps, gen, skip=None):
    for i, p in enumerate(ps):
        p.grad = None if i == skip else (p.detach().float() * 0.5 + torch.randn(p.shape, generator=gen) * 1e-2).to(p.dtype)
    opt.step()


def test_the_optimizer_follows_the_emulation(emu_ops):
    """per group lr / weight decay, fp32 states below min_8bit_size, a parameter without a gradient keeps its step"""
    ws = _weights(0)
    opt, ps = _optimizer(ws)
    hp = [dict(lr=1e-3, weight_decay=1e-2)] * 4 + [dict(lr=2e-3, weight_decay=0.0)] * 2
    ref = [w.clone() for w in ws]
    states = [A.init_state(w) for w in ws]
    g1, g2 = torch.Generator().manual_seed(1), torch.Generator().manual_seed(1)
    for k in range(4):
        skip = 1 if k == 2 else None
        _step(opt, ps, g1, skip)
        for i, w in enumerate(ref):
            if i != skip:
                g = (w.float() * 0.5 + torch.randn(w.shape, generator=g2) * 1e-2).to(w.dtype)
                ref[i] = A.step_emulated(w, g, states[i], **hp[i])
        assert all(torch.equal(_bits(a.detach()), _bits(b)) for a, b in zip(ps, ref))
    assert [opt.state[p]['step'] for p in ps] == [4, 3, 4, 4, 4, 4]
    assert [opt.state[p]['state1'].dtype for p in ps] == [torch.uint8, torch.float32, torch.uint8, torch.uint8,
                                                          torch.float32, torch.uint8]
    m1 = [opt.state[p]['qmap1'] for p in ps if 'qmap1' in opt.state[p]]
    assert all(m is m1[0] for m in m1)                                     # one map per device, as in bnb


def test_state_dict_keeps_every_dtype_and_resumes(emu_ops):
    ws = _weights(2)
    opt, ps = _optimizer(ws)
    g = torch.Generator().manual_seed(7)
    for _ in range(3):
        _step(opt, ps, g)
    sd = opt.state_dict()
    assert set(sd['state'][0]) == {'step', 'state1', 'state2', 'qmap1', 'qmap2', 'absmax1', 'absmax2'}
    assert set(sd['state'][1]) == {'step', 'state1', 'state2'}
    opt2, ps2 = _optimizer([p.detach() for p in ps])
    opt2.load_state_dict(copy.deepcopy(sd))
    for p, p2 in zip(ps, ps2):
        a, b = opt.state[p], opt2.state[p2]
        assert set(a) == set(b) and a['step'] == b['step']
        for k in a:
            if torch.is_tensor(a[k]):
                assert b[k].dtype == a[k].dtype and torch.equal(b[k], a[k]), k
    m1 = [opt2.state[p]['qmap1'] for p in ps2 if 'qmap1' in opt2.state[p]]
    assert all(m is m1[0] for m in m1)
    gens = [torch.Generator().manual_seed(9) for _ in range(2)]
    for _ in range(2):
        _step(opt, ps, gens[0])
        _step(opt2, ps2, gens[1])
    assert all(torch.equal(_bits(a.detach()), _bits(b.detach())) for a, b in zip(ps, ps2))


class _Model:
    def get_param_groups(self, params):
        return [{'params': params}]


@pytest.mark.parametrize('typ', ['AdamW8bit', 'adamw8bit'])
def test_factory_builds_adamw8bit_with_bnbs_defaults(typ):
    import train as T
    from diffusion_pipe_b200 import optim
    ps = [torch.nn.Parameter(torch.zeros(64, 96, dtype=BF16)), torch.nn.Parameter(torch.zeros(96, dtype=BF16))]
    opt = T.make_optimizer_factory({'optimizer': {'type': typ, 'lr': 2e-5}}, _Model())(ps)
    assert isinstance(opt, optim.AdamW8bit)
    g0, g1 = opt.param_groups
    assert (g0['lr'], g0['betas'], g0['eps'], g0['weight_decay'], g1['weight_decay']) == (2e-5, (0.9, 0.999), 1e-8, 1e-2, 0)
    assert opt.min_8bit_size == 4096
    d = optim.AdamW8bit([torch.nn.Parameter(torch.zeros(4))])
    assert d.defaults == dict(lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2)
    opt = T.make_optimizer_factory({'optimizer': {'type': typ, 'lr': 1e-4, 'betas': [0.9, 0.99], 'min_8bit_size': 16,
                                                  'optim_bits': 8, 'weight_decay': 0.1}}, _Model())(ps)
    assert opt.min_8bit_size == 16 and opt.param_groups[0]['betas'] == (0.9, 0.99)


def test_refused_options():
    import train as T
    from diffusion_pipe_b200 import optim
    p = torch.nn.Parameter(torch.zeros(64, 64, dtype=BF16))
    for kw in (dict(block_wise=False), dict(percentile_clipping=5), dict(amsgrad=True), dict(is_paged=True),
               dict(gradient_release=True)):
        with pytest.raises(NotImplementedError):
            optim.AdamW8bit([p], **kw)
    with pytest.raises(NotImplementedError):
        T.make_optimizer_factory({'optimizer': {'type': 'adamw8bit', 'gradient_release': True}}, _Model())([p])
    with pytest.raises(TypeError):
        optim.AdamW8bit([p], not_an_option=1)
    for dt in (torch.float16, torch.float8_e4m3fn):
        with pytest.raises(TypeError):
            optim.AdamW8bit([torch.nn.Parameter(torch.zeros(4, 4).to(dt), requires_grad=False)])
    for q in (p, torch.nn.Parameter(torch.zeros(5, dtype=torch.float32))):      # 8-bit and 32-bit states
        opt = optim.AdamW8bit([q])
        q.grad = torch.ones_like(q)
        with pytest.raises(TypeError, match='CUDA'):
            opt.step()


def test_cli_run_trains_saves_and_resumes(tmp_path, monkeypatch, emu_ops):
    """train.py on a small Flux model with the kernel doubles: 2 steps, a checkpoint, and a resume that runs step 3"""
    import kernel_doubles
    import train as T
    from diffusion_pipe_b200 import ops
    kernel_doubles.install(monkeypatch, ops)
    ds = tmp_path / 'ds.toml'
    ds.write_text("[synthetic]\nnum_examples = 8\nresolution = 128\ntext_len = 32\nt5_dim = 64\nclip_dim = 32\n")

    def cfg(name, max_steps):
        p = tmp_path / f'{name}.toml'
        p.write_text(f"""
output_dir = '{tmp_path}/{name}'
dataset = '{ds}'
epochs = 1
micro_batch_size_per_gpu = 1
gradient_accumulation_steps = 2
save_every_n_steps = 2
max_steps = {max_steps}
eval_before_first_step = false
[model]
type = 'flux'
dtype = 'bfloat16'
device = 'cpu'
transformer_config = {{ num_attention_heads = 2, num_layers = 1, num_single_layers = 1, joint_attention_dim = 64, pooled_projection_dim = 32 }}
[optimizer]
type = 'AdamW8bit'
lr = 1e-3
weight_decay = 0.01
""")
        return p

    def losses(run_dir):
        lines = [json.loads(line) for line in open(os.path.join(run_dir, 'metrics.jsonl'))]
        return [(line['x'], line['value']) for line in lines if line['tag'] == 'train/loss']
    c = cfg('run', 2)
    run_dir = T.main(['--config', str(c)])
    assert os.path.exists(os.path.join(run_dir, 'latest'))
    c.write_text(c.read_text().replace('max_steps = 2', 'max_steps = 3'))
    assert T.main(['--config', str(c), '--resume_from_checkpoint']) == run_dir
    got = losses(run_dir)
    assert [x for x, _ in got] == [1, 2, 3] and all(v == v and v < 100 for _, v in got)


# ---------------------------------------------------------------------------------------------------------------------
# C ABI
# ---------------------------------------------------------------------------------------------------------------------
def test_abi_struct_matches_the_c_compiler(tmp_path):
    from diffusion_pipe_b200 import _abi
    name, cls = 'dpipe_adamw8bit_tensor', _abi.Adamw8bitTensor
    src = '#include <stdio.h>\n#include <stddef.h>\n#include "dpipe.h"\nint main(void){\n'
    for f, _ in cls._fields_:
        src += f'  printf("{f} %zu\\n", offsetof({name}, {f}));\n'
    src += f'  printf("__size__ %zu\\n", sizeof({name}));\n  return 0; }}\n'
    (tmp_path / 'off.c').write_text(src)
    subprocess.run(['gcc', '-std=c99', '-I', os.path.join(ROOT, 'include'), str(tmp_path / 'off.c'), '-o',
                    str(tmp_path / 'off')], check=True)
    out = subprocess.run([str(tmp_path / 'off')], check=True, capture_output=True, text=True).stdout.split()
    got = {out[i]: int(out[i + 1]) for i in range(0, len(out), 2)}
    assert all(getattr(cls, f).offset == got[f] for f, _ in cls._fields_)
    assert ctypes.sizeof(cls) == got['__size__'] == 80


def test_entry_point_rejects_bad_arguments_before_any_cuda_call():
    from diffusion_pipe_b200 import _abi, _lib
    lib = _lib.lib()
    t = (_abi.Adamw8bitTensor * 1)()
    for f in ('p', 'g', 'state1', 'state2', 'absmax1', 'absmax2'):
        setattr(t[0], f, ctypes.c_void_p(16))
    t[0].numel, t[0].dtype = 4096, 0
    maps = ctypes.c_void_p(1024)
    for bad in (dict(dtype=2), dict(numel=-1), dict(g=None), dict(state2=None), dict(absmax2=None)):
        a = (_abi.Adamw8bitTensor * 1)()
        ctypes.memmove(a, t, ctypes.sizeof(t))
        for k, v in bad.items():
            setattr(a[0], k, v)
        assert lib.dpipe_adamw8bit_step(a, 1, maps, maps, None) < 0, bad
        assert b'dpipe_adamw8bit_step' in lib.dpipe_last_error()
    assert lib.dpipe_adamw8bit_step(t, 1, None, maps, None) < 0 and b'maps' in lib.dpipe_last_error()
    assert lib.dpipe_adamw8bit_step(t, -1, maps, maps, None) < 0
    assert lib.dpipe_adamw8bit_step(None, 1, maps, maps, None) < 0
    assert lib.dpipe_adamw8bit_step(None, 0, None, None, None) == 0                  # nothing to do
