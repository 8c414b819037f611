"""GPU: the fused AdamW step kernel (csrc/step_tail.cu adamw_step_multi_kernel) is bit-identical to its specification,
oracle/optim_ref.py adamw_step_emulated, run on CPU copies of the same tensors — at odd sizes, at views 1-7 elements into
a buffer (guard bands untouched), past 64 tensors per call, for mixed bf16 / fp32 lists, with and without weight decay,
with fully decoupled weight decay, at steps 1 and 1000 — and repeatable bit for bit.  Then a small Flux model trained with
`type = 'adamw_optimi'` and gradient clipping through the engine takes every step with the kernel's bits."""
import os
import sys

import pytest
import torch

from oracle import optim_ref as O

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
GUARD = 16


def _bits(t):
    return t.view(torch.int16) if t.dtype == BF16 else t.view(torch.int32)


def _make_set(n, dtype, kahan, offsets, gen):
    """(p, g, m, v, c) as views `offsets[k]` elements into CUDA buffers with GUARD elements after them"""
    vals = [torch.randn(n, generator=gen) * 0.02, torch.randn(n, generator=gen) * 1e-2,
            torch.randn(n, generator=gen) * 3e-3, torch.rand(n, generator=gen) * 1e-4 + 1e-6,
            torch.randn(n, generator=gen) * 1e-6]
    bufs, views = [], []
    for k, val in enumerate(vals):
        if k == 4 and not kahan:
            bufs.append(None)
            views.append(None)
            continue
        off = offsets[k]
        buf = (torch.randn(off + n + GUARD, generator=gen) * 7.0).to(dtype).cuda()
        view = buf[off:off + n]
        view.copy_(val.to(dtype))
        bufs.append(buf)
        views.append(view)
    return bufs, views


def _check_sets(sets, sc):
    """run the kernel over all sets in one call and the emulated oracle on CPU copies; compare bits and guard bands"""
    from diffusion_pipe_b200 import ops
    want = []
    for bufs, views in sets:
        cpu = [v.cpu() if v is not None else None for v in views]
        want.append(O.adamw_step_emulated(*cpu, **sc))
    before = [[b.cpu() if b is not None else None for b in bufs] for bufs, _ in sets]
    ops.adamw_step(*[[views[k] for _, views in sets] for k in range(5)], **sc)
    torch.cuda.synchronize()
    for (bufs, views), w, b0 in zip(sets, want, before):
        for k, got in zip((0, 2, 3, 4), w):
            if got is None:
                continue
            assert torch.equal(_bits(views[k].cpu()), _bits(got)), (k, views[k].numel(), views[k].dtype)
        for k, (buf, view) in enumerate(zip(bufs, views)):
            if buf is None:
                continue
            off = view.data_ptr() - buf.data_ptr()
            off //= buf.element_size()
            n = view.numel()
            host = buf.cpu()
            assert torch.equal(_bits(host[:off]), _bits(b0[k][:off])) and torch.equal(_bits(host[off + n:]), _bits(b0[k][off + n:]))


SCALARS = {
    'step1_wd': dict(lr=2e-5, betas=(0.9, 0.99), weight_decay=1e-2, eps=1e-6, step=1),
    'step1000_wd': dict(lr=3e-4, betas=(0.9, 0.99), weight_decay=1e-1, eps=1e-6, step=1000),
    'step1000_nowd': dict(lr=1e-4, betas=(0.9, 0.999), weight_decay=0.0, eps=1e-8, step=1000),
    'decouple_lr': dict(lr=5e-5, betas=(0.9, 0.99), weight_decay=1e-2, eps=1e-6, step=7, decouple_lr=True, max_lr=1e-4),
}


@pytest.mark.parametrize('case', sorted(SCALARS))
@pytest.mark.parametrize('dtype,kahan', [(BF16, True), (BF16, False), (torch.float32, False)])
def test_kernel_is_bit_identical_to_the_emulated_oracle(case, dtype, kahan):
    sc = O.optimi_scalars(**SCALARS[case])
    gen = torch.Generator().manual_seed(11)
    sets = []
    for n in (1, 7, 8, 9, 4095, (1 << 20) + 3):
        for offsets in ((0, 0, 0, 0, 0), (3, 3, 3, 3, 3), (1, 1, 0, 0, 0), (7, 7, 5, 2, 6)):
            sets.append(_make_set(n, dtype, kahan, offsets, gen))
    _check_sets(sets, sc)


def test_more_than_64_mixed_tensors_in_one_call():
    sc = O.optimi_scalars(lr=1e-4, betas=(0.9, 0.99), weight_decay=1e-2, eps=1e-6, step=3)
    gen = torch.Generator().manual_seed(5)
    sets = []
    for i in range(150):
        dtype, kahan = [(BF16, True), (BF16, False), (torch.float32, False)][i % 3]
        n = [1, 9, 513, 4097, 70001][i % 5]
        off = i % 8
        sets.append(_make_set(n, dtype, kahan, (off, off, off, off, off) if i % 2 else (off, 0, 0, 0, 0), gen))
    _check_sets(sets, sc)


def test_two_runs_give_equal_bits():
    from diffusion_pipe_b200 import ops
    sc = O.optimi_scalars(lr=1e-4, betas=(0.9, 0.99), weight_decay=1e-2, eps=1e-6, step=2)
    outs = []
    for _ in range(2):
        gen = torch.Generator().manual_seed(9)
        sets = [_make_set(n, BF16, True, (off,) * 5, gen) for n, off in ((1 << 22, 0), (12345, 3))]
        ops.adamw_step(*[[views[k] for _, views in sets] for k in range(5)], **sc)
        outs.append([_bits(v.cpu()) for _, views in sets for v in views])
    assert all(torch.equal(a, b) for a, b in zip(*outs))


def test_flux_engine_steps_with_the_kernels_bits():
    """the small Flux model of test_flux_e2e_gpu.py, 3 optimizer steps with `adamw_optimi` and clipping through
    engine.train_batch: before each kernel launch the emulated oracle runs on CPU copies of every (p, g, m, v, c), and the
    kernel's results must equal it bit for bit — so the parameters after 3 steps are those of the run in which every step
    is the emulated oracle"""
    import train as T
    from diffusion_pipe_b200 import ops
    from diffusion_pipe_b200.pipe import ManualPipelineModule, initialize
    from test_flux_e2e_gpu import _batch, _make
    model, _ = _make(3)
    pm = ManualPipelineModule(layers=model.to_layers(), num_stages=1, partition_method='parameters',
                              manual_partition_split=None, loss_fn=model.get_loss_fn(), dynamic_shape=True)
    engine, _, _, _ = initialize(model=pm, config={'train_micro_batch_size_per_gpu': 1, 'gradient_accumulation_steps': 2,
                                                   'gradient_clipping': 1.0, 'steps_per_print': 0})
    params = [p for p in pm.parameters() if p.requires_grad]
    cfg = {'optimizer': {'type': 'adamw_optimi', 'lr': 1e-3, 'weight_decay': 1e-2}}
    engine._configure_optimizer(T.make_optimizer_factory(cfg, model), params)
    real = ops.adamw_step
    checked = []

    def checking(ps, gs, ms, vs, cs, **sc):
        want = [O.adamw_step_emulated(p.cpu(), g.cpu(), m.cpu(), v.cpu(), c.cpu() if c is not None else None, **sc)
                for p, g, m, v, c in zip(ps, gs, ms, vs, cs)]
        real(ps, gs, ms, vs, cs, **sc)
        for w, got in zip(want, zip(ps, ms, vs, cs)):
            for a, b in zip(w, got):
                if a is not None:
                    assert torch.equal(_bits(a), _bits(b.cpu()))
        checked.append(len(ps))
    ops.adamw_step = checking
    try:
        for s in range(3):
            loss = engine.train_batch(iter([_batch(1, 10 * s + i) for i in range(2)]))
            assert torch.isfinite(loss)
    finally:
        ops.adamw_step = real
    assert sum(checked) == 3 * len(params)
    assert any('kahan_comp' in st for st in engine.optimizer.state.values())
    assert float(engine._grad_norm) > 0
