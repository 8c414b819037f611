"""CPU: LoRA on the Wan attention block (wan.WanBlockFn over lora.LoraSite sites) on the kernel test doubles against the oracle with
PEFT-style adapters; the real kernels are exercised by tests/test_wan_gpu.py::test_wan_lora_matches_oracle."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

CFG = {'dim': 256, 'ffn_dim': 512, 'num_heads': 2, 'num_layers': 2, 'text_dim': 64, 'text_len': 16}
RANK = 16


@pytest.fixture
def doubles(monkeypatch):
    import kernel_doubles
    from diffusion_pipe_b200 import ops
    kernel_doubles.install(monkeypatch, ops)
    return ops


def make_pair(device='cpu', transformer_dtype=None):
    from synth import fill_parameters
    from diffusion_pipe_b200.wan import WanPipeline
    from oracle import lora_ref
    from oracle import wan_ref as W
    mc = {'dtype': 'bfloat16', 'device': device, 'transformer_config': CFG}
    if transformer_dtype:
        mc['transformer_dtype'] = transformer_dtype
    model = WanPipeline({'model': mc})
    ref = fill_parameters(W.RefWanModel(dim=256, ffn_dim=512, num_heads=2, num_layers=2, text_dim=64, text_len=16))
    sd = ref.state_dict()
    with torch.no_grad():
        for n, p in model.transformer.named_parameters():
            p.copy_(sd[n].to(p.dtype))
    model.configure_adapter({'type': 'lora', 'rank': RANK, 'alpha': RANK, 'dropout': 0.0})
    lora_ref.add_lora(ref, RANK)
    ref.set_emulate_bf16(True)
    g = torch.Generator().manual_seed(4)
    rp = dict(ref.named_parameters())
    n = 0
    with torch.no_grad():
        for name, p in model.transformer.named_parameters():
            if '.lora_A.' in name or '.lora_B.' in name:
                v = (0.05 * torch.randn(p.shape, generator=g)).bfloat16()
                p.copy_(v)
                rp[name].copy_(v.float())
                n += 1
    assert n == 2 * 10 * 2                       # ten Linear per block, A and B, two blocks
    return model, ref


def make_batch(seed=1):
    from oracle import wan_ref as W
    g = torch.Generator().manual_seed(seed)
    latents, noise = torch.randn(2, 16, 2, 8, 8, generator=g), torch.randn(2, 16, 2, 8, 8, generator=g)
    text = torch.randn(2, 16, 64, generator=g).bfloat16().float()
    t = torch.sigmoid(torch.randn(2, generator=g))
    feats, (target, _) = W.prepare_inputs(latents, text, torch.tensor([10, 16]), t, noise)
    return feats, (target, torch.tensor([]))


def run_both(model, ref, feats, label, dev=None):
    from oracle import flux_ref as R
    from oracle import wan_ref as W
    x = tuple(f.clone().to(dev) if dev else f.clone() for f in feats)
    for layer in model.to_layers():
        x = layer(x)
    loss = model.get_loss_fn()(x, tuple(l.to(dev) if dev else l for l in label))
    loss.backward()
    y = tuple(f.clone() for f in feats)
    for layer in W.to_layers(ref):
        y = layer(y)
    rloss = R.loss_fn(y, label)
    rloss.backward()
    return loss, rloss


def check(model, ref, loss, rloss):
    assert abs(loss.item() - rloss.item()) / abs(rloss.item()) <= 1e-3, (loss.item(), rloss.item())
    rg = {n: p.grad for n, p in ref.named_parameters()}
    seen = 0
    for n, p in model.transformer.named_parameters():
        if not p.requires_grad:
            assert p.grad is None, n
            continue
        assert '.lora_' in n and p.grad is not None, n
        rel = ((p.grad.float().cpu() - rg[n]).norm() / (rg[n].norm() + 1e-12)).item()
        assert rel <= 6e-2, (n, rel)
        seen += 1
    assert seen == 40


def test_wan_lora_forward_backward_matches_oracle(doubles):
    model, ref = make_pair()
    mine = {n: tuple(p.shape) for n, p in model.transformer.named_parameters()}
    assert mine == {n: tuple(p.shape) for n, p in ref.named_parameters()}
    assert all(p.original_name == n for n, p in model.transformer.named_parameters())
    loss, rloss = run_both(model, ref, *make_batch())
    check(model, ref, loss, rloss)
