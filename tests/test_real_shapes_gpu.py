"""GPU: ONE transformer block of every BASELINE.json model at the model's OWN shape against the CPU oracle.

    Flux-dev 1024^2     double + single block   D = 3072, 24 heads x 128, 4096 image + 512 text tokens     (configs[1], [2])
    Qwen-Image 1024^2   double-stream block     D = 3072, 24 heads, 4096 image + 256 text tokens, biased projections (configs[4])
    Wan2.1-14B          attention block         D = 5120, 40 heads, FFN 13824, 2048 video + 512 text tokens (configs[3]; the
                                                 model's width / heads / FFN, a quarter of the 33-frame sequence so that the
                                                 fp32 oracle's 40-head score tensors stay within host memory and minutes)

The small-shape tests next door (D = 256, 2 heads) cannot see an indexing mistake that only shows at 24 or 40 heads (the QKV
epilogue's head arithmetic, the 12 / 20 N-tiles a LayerNorm row or a full-width RMSNorm spans, GEMM tile tails at
N = 21504 / 13824).  Here the outputs, the gradients w.r.t. every block input, a scalar loss and EVERY parameter gradient are
compared on identical inputs and weights (weights ~ N(0, 0.02) as in bench.py, biases and norm scales perturbed).

Tolerances (north star: loss within 1e-3 relative; bf16 kernels with fp32 accumulation vs the oracle):
    loss                                  <= 1e-3 relative  (oracle with the reference's bf16 rounding points emulated)
    outputs / input gradients             <= 1.5e-2 relative Frobenius (emulated), <= 2e-2 (fp32 oracle)
    parameter gradients                   <= 2e-2 relative Frobenius for every weight matrix (emulated oracle); 5e-2 for the
                                          vectors (biases, norm scales: column reductions whose true value is often near zero,
                                          e.g. a key bias under a shift-invariant softmax)
The oracle runs on the host cores of the GPU box (about 20-60 s per block and mode)."""
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))


def _rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-12)).item()


def _perturb(blk, seed):
    """biases / norm scales away from their 0 / 1 initial values so that their gradients and index arithmetic matter"""
    dev = next(blk.parameters()).device
    g = torch.Generator(device=dev).manual_seed(seed)
    with torch.no_grad():
        for n, p in blk.named_parameters():
            if p.dim() == 1 or n.endswith('modulation'):
                noise = torch.randn(p.shape, generator=g, device=dev, dtype=torch.float32)
                if 'norm' in n and n.endswith('weight'):
                    p.copy_((1 + 0.1 * noise).to(p.dtype))
                elif n.endswith('modulation'):
                    pass
                else:
                    p.copy_((0.05 * noise).to(p.dtype))


def _load(ref, blk):
    sd = {k: v.detach().float().cpu() for k, v in blk.state_dict().items()}
    missing, unexpected = ref.load_state_dict(sd, strict=False)
    assert not missing and not unexpected, (missing[:4], unexpected[:4])


def _set_emulate(ref, emu):
    for m in ref.modules():
        if hasattr(m, 'emulate_bf16'):
            m.emulate_bf16 = emu


def _compare(blk, ref, run_product, run_oracle, n_out, modes=((True, 1.5e-2), (False, 2e-2)), grad_tol=2e-2):
    """run_*() -> (tuple of outputs and input gradients, loss float); the product's parameter gradients are read from
    blk.named_parameters(), the oracle's from ref.named_parameters()"""
    got, loss = run_product()
    if torch.cuda.is_available():
        torch.cuda.synchronize()
    pg = {n: p.grad.detach().float().cpu() for n, p in blk.named_parameters() if p.grad is not None}
    report = {}
    for emu, tol in modes:
        _set_emulate(ref, emu)
        ref.zero_grad()
        want, rloss = run_oracle()
        for i, (a, b) in enumerate(zip(got, want)):
            r = _rel(a, b)
            report[(emu, i)] = r
            assert r <= tol, (emu, 'output' if i < n_out else 'input gradient', i, r, report)
        lrel = abs(loss - rloss) / abs(rloss)
        assert lrel <= (1e-3 if emu else 5e-3), (emu, loss, rloss, lrel)
        if emu or len(modes) == 1:
            rg = {n: p.grad.detach().float() for n, p in ref.named_parameters() if p.grad is not None}
            assert set(pg) == set(rg), sorted(set(pg) ^ set(rg))[:6]
            bad = []
            for n in rg:
                r = _rel(pg[n], rg[n])
                lim = 5e-2 if rg[n].numel() <= 16384 else grad_tol
                if r > lim:
                    bad.append((round(r, 4), n))
            assert not bad, sorted(bad, reverse=True)[:8]
    return report


def _flux_rope(Lt, side):
    from oracle import flux_ref as R
    Li = side * side
    ids = torch.zeros(Lt + Li, 3)
    ids[Lt:, 1] = torch.arange(Li) // side
    ids[Lt:, 2] = torch.arange(Li) % side
    return R.flux_rope_tables(ids)


def check_flux(kind, D, H, Lt, side, dev='cuda', batch=1):
    from diffusion_pipe_b200 import flux_blocks as FB
    from oracle import flux_ref as R
    Li = side * side
    torch.manual_seed(21)
    if kind == 'double':
        blk, ref = FB.FluxTransformerBlock(D, H, device=dev), R.RefFluxTransformerBlock(D, H)
    else:
        blk, ref = FB.FluxSingleTransformerBlock(D, H, device=dev), R.RefFluxSingleTransformerBlock(D, H)
    _perturb(blk, 5)
    _load(ref, blk)
    cos, sin = _flux_rope(Lt, side)
    g = torch.Generator().manual_seed(3)
    hid, enc = torch.randn(batch, Li, D, generator=g).bfloat16(), torch.randn(batch, Lt, D, generator=g).bfloat16()
    temb = torch.randn(batch, D, generator=g).bfloat16()   # a different modulation row per sample
    t_h, t_e = torch.randn(batch, Li, D, generator=g).bfloat16(), torch.randn(batch, Lt, D, generator=g).bfloat16()

    def run(block, dev, dtype):
        h = hid.detach().clone().to(dev, dtype).requires_grad_(True)
        e = enc.detach().clone().to(dev, dtype).requires_grad_(True)
        t = temb.detach().clone().to(dev, dtype).requires_grad_(True)
        eo, ho = block(h, e, t, (cos.to(dev), sin.to(dev)))
        # an MSE against a fixed target: what the pipeline's last layer puts behind the blocks (models/base.py:418-436)
        loss = ((ho.float() - t_h.to(dev).float()) ** 2).mean() + ((eo.float() - t_e.to(dev).float()) ** 2).mean()
        (loss * 4096.0).backward()
        return (ho.detach(), eo.detach(), h.grad, e.grad, t.grad), loss.item()
    return _compare(blk, ref, lambda: run(blk, dev, torch.bfloat16), lambda: run(ref, 'cpu', torch.float32), n_out=2)


@pytest.mark.parametrize('kind', ['double', 'single'])
def test_flux_dev_block_at_1024px(kind):
    """models/flux.py:497-533 over diffusers' Flux blocks at configs/flux_dev_config.json shapes"""
    check_flux(kind, D=3072, H=24, Lt=512, side=64)


@pytest.mark.parametrize('kind', ['double', 'single'])
def test_flux_block_at_micro_batch_3(kind):
    """three samples with their own temb at the Flux width and head count, short sequence: the per-sample gate of
    EPI_GATE_RES, the batch index of the QKV epilogue and the 3-4 sample modulation backward inside real blocks"""
    check_flux(kind, D=3072, H=24, Lt=128, side=32, batch=3)


def check_qwen(D, H, Lt, side, dev='cuda', batch=1):
    from diffusion_pipe_b200 import qwen_image as QI
    from oracle import qwen_ref as Q
    Li = side * side
    torch.manual_seed(22)
    blk, ref = QI.QwenImageTransformerBlock(D, H, device=dev), Q.RefQwenImageTransformerBlock(D, H)
    _perturb(blk, 6)
    _load(ref, blk)
    vc, vs, tc, ts = Q.qwen_rope_tables([(1, side, side)], Lt)
    vid, txt = torch.stack([vc, vs]), torch.stack([tc, ts])          # [2, L, 128] each (cos, sin)
    joint = torch.cat([txt, vid], dim=1)
    g = torch.Generator().manual_seed(4)
    hid, enc = torch.randn(batch, Li, D, generator=g).bfloat16(), torch.randn(batch, Lt, D, generator=g).bfloat16()
    temb = torch.randn(batch, D, generator=g).bfloat16()
    t_h, t_e = torch.randn(batch, Li, D, generator=g).bfloat16(), torch.randn(batch, Lt, D, generator=g).bfloat16()

    def finish(eo, ho, h, e, t, dev):
        loss = ((ho.float() - t_h.to(dev).float()) ** 2).mean() + ((eo.float() - t_e.to(dev).float()) ** 2).mean()
        (loss * 4096.0).backward()
        return (ho.detach(), eo.detach(), h.grad, e.grad, t.grad), loss.item()

    def run_product():
        h, e, t = (x.detach().clone().to(dev).requires_grad_(True) for x in (hid, enc, temb))
        eo, ho = blk(hidden_states=h, encoder_hidden_states=e, temb=t,
                     image_rotary_emb=(joint[0].to(dev).contiguous(), joint[1].to(dev).contiguous()))
        return finish(eo, ho, h, e, t, dev)

    def run_oracle():
        h, e, t = (x.detach().float().requires_grad_(True) for x in (hid, enc, temb))
        eo, ho = ref(h, e, t, ((vid[0], vid[1]), (txt[0], txt[1])), None)
        return finish(eo, ho, h, e, t, 'cpu')
    return _compare(blk, ref, run_product, run_oracle, n_out=2)


def test_qwen_image_block_at_1024px():
    """models/qwen_image.py:519-605 + QwenDoubleStreamAttnProcessor2_0 (:91-174): biased q/k/v, separate image / text rope"""
    check_qwen(D=3072, H=24, Lt=256, side=64)


def test_qwen_image_block_at_micro_batch_3():
    check_qwen(D=3072, H=24, Lt=128, side=32, batch=3)


def check_wan(D, F, H, Lc, grid, dev='cuda'):
    from diffusion_pipe_b200 import wan as WN
    from oracle import wan_ref as W
    L = grid[0] * grid[1] * grid[2]
    torch.manual_seed(23)
    blk, ref = WN.WanAttentionBlock(D, F, H, device=dev), W.RefWanAttentionBlock(D, F, H)
    _perturb(blk, 7)
    _load(ref, blk)
    cos, sin = W.wan_rope_tables(grid)
    g = torch.Generator().manual_seed(5)
    x0 = torch.randn(1, L, D, generator=g).bfloat16()
    e0 = (0.3 * torch.randn(1, 1, 6, D, generator=g)).bfloat16()
    ctx = torch.randn(1, Lc, D, generator=g).bfloat16()
    tgt = torch.randn(1, L, D, generator=g).bfloat16()

    def finish(y, x, e, c, dev):
        loss = ((y.float() - tgt.to(dev).float()) ** 2).mean()
        (loss * 4096.0).backward()
        return (y.detach(), x.grad, e.grad, c.grad), loss.item()

    def run_product():
        x, e, c = (t.detach().clone().to(dev).requires_grad_(True) for t in (x0, e0, ctx))
        seq_lens = torch.full((1,), L, dtype=torch.long, device=dev)
        grid_sizes = torch.tensor([grid], dtype=torch.long, device=dev)
        y = blk(x, e, seq_lens, grid_sizes, (cos.to(dev).contiguous(), sin.to(dev).contiguous()), c, None)
        return finish(y, x, e, c, dev)

    def run_oracle():
        x, e, c = (t.detach().float().requires_grad_(True) for t in (x0, e0, ctx))
        y = ref(x, e, [L], cos, sin, c, None)
        return finish(y, x, e, c, 'cpu')
    return _compare(blk, ref, run_product, run_oracle, n_out=1)


def test_wan_14b_block():
    """models/wan/wan.py:521-529 -> WanAttentionBlock (models/wan/model.py:277-312) at the 14B width: full-width (5120)
    RMSNorm on q / k, 3-axis rope, 40 heads, cross-attention over all 512 text slots, FFN 13824"""
    check_wan(D=5120, F=13824, H=40, Lc=512, grid=(2, 32, 32))
