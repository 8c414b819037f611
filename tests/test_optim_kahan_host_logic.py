"""CPU: optimi's AdamW with Kahan-summed bf16 weights (`type = 'adamw_optimi'`) — the kernel's specification against the
recalled optimi text, the Kahan property itself, the optimizer factory, the optimizer's state through the engine's
checkpoints and LR schedulers (with `ops.adamw_step` replaced by the emulated oracle inside this file only), and the C
entry point's argument checks."""
import ctypes
import os
import socket
import sys

import pytest
import torch
from torch import nn

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (ROOT, HERE):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from oracle import optim_ref as O  # noqa: E402

BF16 = torch.bfloat16


def _ulp_bf16(x):
    """bf16 ulp of |x| (fp64), normal range"""
    e = torch.floor(torch.log2(x.abs().double().clamp_min(2.0 ** -126)))
    return torch.pow(2.0, e - 7)


def _random_state(n, seed, dtype=BF16):
    g = torch.Generator().manual_seed(seed)
    p = (torch.randn(n, generator=g) * 0.02).to(dtype)
    grad = (torch.randn(n, generator=g) * 1e-2).to(dtype)
    m = (torch.randn(n, generator=g) * 3e-3).to(dtype)
    v = (torch.rand(n, generator=g) * 1e-4 + 1e-6).to(dtype)
    c = (torch.randn(n, generator=g) * 1e-6).to(dtype) if dtype == BF16 else None
    return p, grad, m, v, c


@pytest.mark.parametrize('step', [1, 2, 10, 1000])
def test_torch_ops_text_and_emulated_specification_agree(step):
    """one step from random states: the recalled optimi text (bf16 torch ops) and the kernel's specification differ only
    where torch contracts a multiply-add, by at most one bf16 ulp of that op's operands or result"""
    n = 1 << 18
    p, g, m, v, c = _random_state(n, step)
    sc = O.optimi_scalars(2e-5, (0.9, 0.99), 1e-2, 1e-6, step)
    tp, tm, tv, tc = O.optimi_adamw_torch_ops(p, g, m, v, c, **sc)
    ep, em, ev, ec = O.adamw_step_emulated(p, g, m, v, c, **sc)
    assert (tp.float() - ep.float()).abs().le(_ulp_bf16(ep.float()).float()).all()
    upd = O.update_fp32(em, ev, lr=sc['lr'], eps=sc['eps']).double()
    operands = {
        'm': (tm, em, torch.maximum(m.double().abs(), g.double().abs())),
        'v': (tv, ev, torch.maximum(v.double().abs(), g.double().square())),
        'c': (tc, ec, torch.maximum(c.double().abs(), upd.abs())),
        'p': (tp, ep, torch.maximum(p.double().abs(), ec.double().abs())),
    }
    for name, (t, e, mag) in operands.items():
        diff = (t.double() - e.double()).abs()
        mag = torch.maximum(mag, e.double().abs())                 # a result that crossed a power of two
        same = (t.view(torch.int16) == e.view(torch.int16)).double().mean().item()
        assert same >= 0.999, (name, same)
        bound = _ulp_bf16(mag)
        if name == 'c':        # torch's CPU bf16 add_(eps) rounds eps to bf16: den may sit one bf16 ulp from the kernel's
            bound = bound + upd.abs() * 2.0 ** -7
        bad = diff > bound
        assert not bad.any(), (name, int(bad.sum()), diff[bad][:4], mag[bad][:4])


def test_kahan_summation_keeps_the_small_updates():
    """lr = 2e-5 for 2000 steps on N(0, 0.02) bf16 weights: with Kahan summation p + c follows the fp64 sum of the
    per-step updates to within one bf16 ulp everywhere; the plain bf16 update leaves most weights where they started.
    (bf16 compensation is not exact: under a gradient of one sign every step its own rounding accumulates, and the error
    grows past one ulp.)"""
    n, steps, lr = 100_000, 2000, 2e-5
    gen = torch.Generator().manual_seed(7)
    p0 = (torch.randn(n, generator=gen) * 0.02).to(BF16)
    drift = torch.randn(n, generator=gen) * 3e-4          # each weight's gradient: a small bias plus step-to-step noise
    zero = torch.zeros(n, dtype=BF16)
    pk, mk, vk, ck = p0.clone(), zero.clone(), zero.clone(), zero.clone()
    pp, mp, vp = p0.clone(), zero.clone(), zero.clone()
    ref = p0.double()
    for t in range(1, steps + 1):
        g = (drift + torch.randn(n, generator=gen) * 1e-3).to(BF16)
        sc = O.optimi_scalars(lr, (0.9, 0.99), 0.0, 1e-6, t)
        pk, mk, vk, ck = O.adamw_step_emulated(pk, g, mk, vk, ck, **sc)
        ref = ref + O.update_fp32(mk, vk, lr=sc['lr'], eps=sc['eps']).double()
        pp, mp, vp, _ = O.adamw_step_emulated(pp, g, mp, vp, None, **sc)
    unit = _ulp_bf16(torch.maximum(ref.abs(), torch.full_like(ref, 2.0 ** -10)))
    err_kahan = ((pk.double() + ck.double()) - ref).abs() / unit
    err_plain = (pp.double() - ref).abs() / unit
    assert err_kahan.max().item() <= 1.0, err_kahan.max().item()
    unchanged = (pp.view(torch.int16) == p0.view(torch.int16)).double().mean().item()
    assert unchanged > 0.5, unchanged
    assert err_plain.median().item() > 10.0, err_plain.median().item()


def test_product_scalars_are_the_fp32_roundings_of_the_recalled_formula():
    from diffusion_pipe_b200 import optim
    for t in (1, 2, 10, 1000):
        for kw in ({}, {'decouple_lr': True, 'max_lr': 1e-4}):
            assert optim.step_scalars(3e-5, (0.9, 0.99), 1e-2, 1e-6, t, **kw) == \
                O.optimi_scalars(3e-5, (0.9, 0.99), 1e-2, 1e-6, t, **kw)
    sc = optim.step_scalars(1e-4, (0.9, 0.99), 1e-2, 1e-6, 1)
    assert sc['beta1_comp'] == 1.0 and sc['beta2_hat'] == 0.0        # step 1: m = g, v = g^2
    assert optim.step_scalars(1e-4, (0.9, 0.99), 0.0, 1e-6, 5)['decay'] == 1.0


def _emulated_adamw_step(params, grads, exp_avgs, exp_avg_sqs, kahan_comps, **sc):
    """ops.adamw_step on CPU tensors: the kernel's specification, written back in place"""
    for p, g, m, v, c in zip(params, grads, exp_avgs, exp_avg_sqs, kahan_comps):
        out = O.adamw_step_emulated(p, g, m, v, c, **sc)
        for dst, src in zip((p, m, v, c), out):
            if dst is not None:
                dst.copy_(src)


@pytest.fixture
def emulated_ops(monkeypatch):
    from diffusion_pipe_b200 import ops
    calls = []

    def fake(*a, **k):
        calls.append(len(a[0]))
        _emulated_adamw_step(*a, **k)
    monkeypatch.setattr(ops, 'adamw_step', fake)
    return calls


class _M:
    def get_param_groups(self, params):
        return [{'params': params}]


def test_optimizer_factory_builds_optimi_adamw(emulated_ops):
    import train as T
    from diffusion_pipe_b200 import optim
    w = nn.Parameter(torch.randn(8, 4).to(BF16))
    b = nn.Parameter(torch.zeros(8, dtype=BF16))
    f = nn.Parameter(torch.randn(3, 3))
    opt = T.make_optimizer_factory({'optimizer': {'type': 'adamw_optimi', 'lr': 1e-4}}, _M())([w, b, f])
    assert isinstance(opt, optim.AdamW)
    g0, g1 = opt.param_groups
    assert g0['betas'] == (0.9, 0.99) and g0['eps'] == 1e-6 and g0['weight_decay'] == 1e-2 and g1['weight_decay'] == 0
    assert g0['params'] == [w, f] and g1['params'] == [b]
    assert g0['kahan_sum'] is None and g0['decouple_lr'] is False and g0['max_lr'] is None
    for p in (w, b, f):
        p.grad = torch.randn_like(p)
    opt.step()
    assert emulated_ops == [2, 1]                                    # one call per param group
    assert set(opt.state[w]) == {'step', 'exp_avg', 'exp_avg_sq', 'kahan_comp'} and opt.state[w]['exp_avg'].dtype == BF16
    assert 'kahan_comp' not in opt.state[f] and opt.state[f]['exp_avg'].dtype == torch.float32
    assert opt.state[w]['step'] == 1
    # the [optimizer] keys of the reference's TOML: betas / beta2_half_life, kahan_sum, decouple_lr, max_lr
    cfg = {'optimizer': {'type': 'adamw_optimi', 'lr': 2e-5, 'betas': [0.9, 0.99], 'weight_decay': 0.01, 'eps': 1e-8,
                         'kahan_sum': False, 'decouple_lr': True, 'beta2_half_life': 64}}
    opt = T.make_optimizer_factory(cfg, _M(), global_batch_size=16)([w, b])
    assert opt.param_groups[0]['betas'] == (0.9, 0.5 ** (16 / 64)) and opt.param_groups[0]['max_lr'] == 2e-5
    w.grad = torch.randn_like(w)
    b.grad = None
    opt.step()
    assert 'kahan_comp' not in opt.state[w] and b not in opt.state
    # `adamw` is still torch's fused AdamW; the types without a kernel still raise
    assert type(T.make_optimizer_factory({'optimizer': {'type': 'adamw', 'lr': 1e-4, 'kahan_sum': True}}, _M())([w])) \
        is torch.optim.AdamW
    for typ in ('stableadamw', 'adamw8bitkahan'):
        with pytest.raises(NotImplementedError):
            T.make_optimizer_factory({'optimizer': {'type': typ, 'lr': 1e-4}}, _M())([w])
    with pytest.raises(TypeError):
        T.make_optimizer_factory({'optimizer': {'type': 'adamw_optimi', 'lr': 1e-4, 'foreach': True}}, _M())([w])
    with pytest.raises(NotImplementedError):
        optim.AdamW([w], lr=1e-4, gradient_release=True)


def test_cpu_parameters_are_refused():
    """the product has no CPU path: the real ops.adamw_step refuses non-CUDA tensors before any library call"""
    from diffusion_pipe_b200 import optim
    w = nn.Parameter(torch.randn(4, 4).to(BF16))
    w.grad = torch.randn_like(w)
    with pytest.raises(TypeError, match='CUDA'):
        optim.AdamW([w], lr=1e-4).step()


# --------------------------------------------------------------------------------------------------------------------
# the optimizer inside the pipeline engine (gloo, one process)
# --------------------------------------------------------------------------------------------------------------------
class _BfLinear(nn.Module):
    """a linear layer with bf16 weights on fp32 activations (its gradients come back bf16)"""

    def __init__(self, d, seed):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        self.weight = nn.Parameter((torch.randn(d, d, generator=g) * 0.02).to(BF16))
        self.bias = nn.Parameter(torch.zeros(d, dtype=BF16))

    def forward(self, x):
        return torch.tanh(x @ self.weight.float().t() + self.bias.float())


class _Fp32Linear(nn.Module):
    def __init__(self, d, seed):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        self.lin = nn.Linear(d, d)
        with torch.no_grad():
            self.lin.weight.copy_(torch.randn(d, d, generator=g) * 0.1)
            self.lin.bias.copy_(torch.randn(d, generator=g) * 0.1)

    def forward(self, x):
        return self.lin(x)


def _layers():
    layers = [_BfLinear(16, 1), _Fp32Linear(16, 2), _BfLinear(16, 3)]
    for li, l in enumerate(layers):
        for n, p in l.named_parameters():
            p.original_name = f'{li}.{n}'
    return layers


def _loss(out, label):
    return ((out - label[0]) ** 2).mean()


def _batches(step, gas=2):
    g = torch.Generator().manual_seed(100 + step)
    return [(torch.randn(4, 16, generator=g), (torch.randn(4, 16, generator=g), torch.tensor([]))) for _ in range(gas)]


def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    return port


@pytest.fixture
def gloo_world_1(monkeypatch):
    monkeypatch.setenv('RANK', '0')
    monkeypatch.setenv('WORLD_SIZE', '1')
    monkeypatch.setenv('MASTER_ADDR', '127.0.0.1')
    monkeypatch.setenv('MASTER_PORT', str(_free_port()))
    from diffusion_pipe_b200.pipe import dist
    dist.init_distributed('gloo')
    yield
    import torch.distributed as tdist
    if tdist.is_initialized():
        tdist.destroy_process_group()


def _engine(sched_factor=None):
    import train as T
    from diffusion_pipe_b200.pipe import ManualPipelineModule, initialize
    pm = ManualPipelineModule(layers=_layers(), num_stages=1, partition_method='uniform', loss_fn=_loss, dynamic_shape=True,
                              device=torch.device('cpu'))
    engine, _, _, _ = initialize(model=pm, config={'train_micro_batch_size_per_gpu': 4, 'gradient_accumulation_steps': 2,
                                                   'gradient_clipping': 1.0, 'steps_per_print': 0, 'stage_link': 'dist'})
    cfg = {'optimizer': {'type': 'adamw_optimi', 'lr': 1e-3, 'weight_decay': 0.1}}
    engine._configure_optimizer(T.make_optimizer_factory(cfg, _M()), [p for p in pm.parameters() if p.requires_grad])
    if sched_factor is not None:
        engine.lr_scheduler = torch.optim.lr_scheduler.LambdaLR(engine.optimizer, sched_factor)
    return engine, pm


def _params(pm):
    return {p.original_name: p.detach().clone() for p in pm.parameters()}


def test_engine_checkpoint_round_trip_continues_bit_identically(gloo_world_1, emulated_ops, tmp_path):
    """stopped, saved and reloaded after step k, training continues with the same bits as a run that never stopped
    (exp_avg, exp_avg_sq, kahan_comp and the host step count all travel through save_checkpoint / load_checkpoint)"""
    k, total = 2, 5
    eng, pm = _engine(lambda s: 0.5 ** s)
    for s in range(total):
        eng.train_batch(iter(_batches(s)))
    want = _params(pm)

    eng, pm = _engine(lambda s: 0.5 ** s)
    for s in range(k):
        eng.train_batch(iter(_batches(s)))
    eng.save_checkpoint(str(tmp_path))
    assert any('kahan_comp' in st for st in eng.optimizer.state_dict()['state'].values())
    eng, pm = _engine(lambda s: 0.5 ** s)
    before = _params(pm)
    eng.load_checkpoint(str(tmp_path))
    assert any(not torch.equal(before[n], p) for n, p in _params(pm).items())
    assert {st['step'] for st in eng.optimizer.state.values()} == {k}
    for s in range(k, total):
        eng.train_batch(iter(_batches(s)))
    got = _params(pm)
    for n in want:
        assert torch.equal(got[n].view(torch.int16) if got[n].dtype == BF16 else got[n],
                           want[n].view(torch.int16) if want[n].dtype == BF16 else want[n]), n


def test_engine_step_follows_the_lr_scheduler(gloo_world_1, monkeypatch):
    """the step reads group['lr'] every time: a scheduler that halves it between steps reaches the kernel's scalars"""
    from diffusion_pipe_b200 import ops
    seen = []

    def fake(*a, **k):
        seen.append((k['lr'], k['decay']))
        _emulated_adamw_step(*a, **k)
    monkeypatch.setattr(ops, 'adamw_step', fake)
    eng, _ = _engine(lambda s: 0.5 ** s)
    for s in range(3):
        eng.train_batch(iter(_batches(s)))
    lrs = sorted({lr for lr, _ in seen}, reverse=True)
    assert lrs == [O.f32(1e-3), O.f32(5e-4), O.f32(2.5e-4)]
    assert O.f32(1 - 2.5e-4 * 0.1) in {d for _, d in seen}


def test_entry_point_refuses_bad_arguments_without_a_gpu():
    from diffusion_pipe_b200 import _lib
    lib = _lib.lib()
    one = (ctypes.c_void_p * 1)(256)
    none = (ctypes.c_void_p * 1)(None)
    numel = (ctypes.c_int64 * 1)(10)
    bf16, fp32, bad = (ctypes.c_int * 1)(0), (ctypes.c_int * 1)(1), (ctypes.c_int * 1)(2)
    sc = (1e-4, 1.0, 0.0, 1.0, 1e-6, 1.0)

    def call(p=one, g=one, m=one, v=one, c=None, numels=numel, dtypes=bf16, n=1):
        return lib.dpipe_adamw_step(p, g, m, v, c, numels, dtypes, n, *sc, None)
    assert call(n=-1) < 0 and b'n < 0' in lib.dpipe_last_error()
    assert call(p=None) < 0 and b'null' in lib.dpipe_last_error()
    for kw in ({'p': none}, {'g': none}, {'m': none}, {'v': none}):
        assert call(**kw) < 0 and b'null pointer' in lib.dpipe_last_error()
    assert call(dtypes=bad) < 0 and b'dtype' in lib.dpipe_last_error()
    assert call(c=one, dtypes=fp32) < 0 and b'bf16 tensors only' in lib.dpipe_last_error()
    assert call(numels=(ctypes.c_int64 * 1)(-3)) < 0 and b'numel' in lib.dpipe_last_error()
    assert call(n=0) == 0 and call(p=none, numels=(ctypes.c_int64 * 1)(0)) == 0     # nothing to do: no device needed
