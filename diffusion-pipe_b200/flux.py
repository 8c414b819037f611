"""Flux model definition on the sm_90a kernels — the drop-in for the reference's models/flux.py.

Same plugin surface (models/base.py:348-445 via models/flux.py:153-548): `FluxPipeline(config)` with `name`,
`checkpointable_layers`, `prepare_inputs(batch, timestep_quantile)`, `to_layers()`, `get_loss_fn()`; the layers speak
the reference's tuple protocol `(hidden_states, encoder_hidden_states, temb, freqs_cos, freqs_sin, img_seq_len)`
(models/flux.py:487,510,533).  What changes is underneath: the transformer is `FluxTransformer2DModel` below, whose
blocks are the fused autograd Functions of flux_blocks.py, instead of diffusers' module tree + autocast + cuBLAS/SDPA.

VAE / text encoders / latent caching are outside the hot path (SURVEY.md section 8) and are not provided here;
`prepare_inputs` consumes the same cached tensors (`latents`, `t5_embed`, `clip_embed`, `mask`) as the reference.
"""
import json
import math
import os
import re

import torch
from torch import nn

from . import ops
from .plugin import PluginSurface
from .flux_blocks import (FluxSingleTransformerBlock, FluxTransformerBlock, _AdaNorm, _acc_vec, _grad_buf, _mod_bwd,
                          _mod_fwd, _plain, _silu_bf16)

NUM_DOUBLE_BLOCKS = 19
NUM_SINGLE_BLOCKS = 38

FLUX_DEV_CONFIG = {   # reference: configs/flux_dev_config.json
    'attention_head_dim': 128, 'num_attention_heads': 24, 'num_layers': 19, 'num_single_layers': 38,
    'in_channels': 64, 'joint_attention_dim': 4096, 'pooled_projection_dim': 768, 'guidance_embeds': True,
    'axes_dims_rope': [16, 56, 56],
}


# =====================================================================================================================
# generic pieces
# =====================================================================================================================
class LinearFn(torch.autograd.Function):
    """y = x W^T + b on the wgmma GEMM; backward = dgrad + wgrad GEMMs + a column-sum kernel."""

    @staticmethod
    def forward(ctx, x, lin):
        shp = x.shape
        x2 = x.reshape(-1, shp[-1])
        if x2.dtype != torch.bfloat16:
            x2 = x2.to(torch.bfloat16)
        if not x2.is_contiguous():
            x2 = x2.contiguous()
        y = ops.gemm(x2, lin.weight, bias=lin.bias, cta_group=2 if x2.shape[0] > 128 else 1)
        ctx.lin = lin
        ctx.save_for_backward(x2)
        ctx.shp = shp
        ctx.in_dtype = x.dtype
        return y.view(*shp[:-1], lin.weight.shape[0])

    @staticmethod
    def backward(ctx, dy):
        lin = ctx.lin
        (x2,) = ctx.saved_tensors
        dy2 = dy.reshape(-1, dy.shape[-1])
        if dy2.dtype != torch.bfloat16:
            dy2 = dy2.to(torch.bfloat16)
        if not dy2.is_contiguous():
            dy2 = dy2.contiguous()
        cg = 2 if x2.shape[0] > 128 else 1
        if lin.weight.requires_grad:
            def wgrad(lin=lin, dy2=dy2, x2=x2, cg=cg):
                g, acc = _grad_buf(lin.weight)
                ops.gemm(dy2, x2, a_mn=True, b_mn=True, out=g, accumulate=acc, cta_group=cg)
                if lin.bias is not None:
                    _acc_vec(lin.bias, ops.colsum(dy2))
            ops.defer(wgrad)
        dx = None
        if ctx.needs_input_grad[0]:
            dx = ops.gemm(dy2, lin.weight, b_mn=True, cta_group=cg).view(ctx.shp).to(ctx.in_dtype)
        return dx, None


def linear(x, lin):
    return LinearFn.apply(x, lin)


class AdaLNContinuousFn(torch.autograd.Function):
    """diffusers AdaLayerNormContinuous(elementwise_affine=False): LN(x) * (1 + scale) + shift with
    (scale, shift) = linear(silu(temb)).chunk(2)  — chunk order per models/flux.py:280-288."""

    @staticmethod
    def forward(ctx, x, temb, lin):
        B, L, D = x.shape
        mod = _mod_fwd(temb, lin)                               # [B, 2D]: scale, shift
        x2 = x.reshape(B * L, D)
        xn, mean, rstd = ops.ln_modulate_fwd(x2, mod[:, 0:D], mod[:, D:2 * D], B, L)
        ctx.lin = lin
        ctx.save_for_backward(x2, temb, mod, mean, rstd)
        ctx.dims = (B, L, D)
        return xn.view(B, L, D)

    @staticmethod
    def backward(ctx, dxn):
        x2, temb, mod, mean, rstd = ctx.saved_tensors
        B, L, D = ctx.dims
        dxn2 = dxn.reshape(B * L, D)
        if dxn2.dtype != torch.bfloat16:
            dxn2 = dxn2.to(torch.bfloat16)
        dmod = torch.empty((B, 2 * D), dtype=torch.float32, device=x2.device)
        dx, part = ops.ln_modulate_bwd(dxn2.contiguous(), x2, mod[:, 0:D], mean, rstd, B, L)
        ops.colreduce_finish(part, per_sample0=dmod[:, 0:D], per_sample1=dmod[:, D:2 * D])
        d_temb = torch.zeros((B, D), dtype=torch.float32, device=x2.device)
        _mod_bwd(dmod, temb, ctx.lin, d_temb)
        return dx.view(B, L, D), d_temb.to(temb.dtype), None


class MseLossFn(torch.autograd.Function):
    """models/base.py:418-436 default loss: mean((output - target)^2 * mask) in fp32."""

    @staticmethod
    def forward(ctx, output, target, mask):
        o = output if output.dtype == torch.bfloat16 else output.to(torch.bfloat16)
        loss, dout = ops.mse_loss(o.contiguous(), target, mask)
        ctx.save_for_backward(dout)
        ctx.shape = output.shape
        ctx.dtype = output.dtype
        return loss

    @staticmethod
    def backward(ctx, g):
        (dout,) = ctx.saved_tensors
        return (dout.float() * g).to(ctx.dtype).view(ctx.shape), None, None


def timestep_sinusoid(t, dim=256, max_period=10000.0):
    """diffusers Timesteps(256, flip_sin_to_cos=True, downscale_freq_shift=0) — [cos | sin], fp32."""
    half = dim // 2
    exponent = -math.log(max_period) * torch.arange(0, half, dtype=torch.float32, device=t.device) / half
    emb = t[:, None].float() * torch.exp(exponent)[None, :]
    return torch.cat([torch.cos(emb), torch.sin(emb)], dim=-1)


def flux_rope_tables(ids, axes_dim=(16, 56, 56), theta=10000.0):
    """diffusers FluxPosEmbed: ids [L, 3] -> (cos, sin) fp32 [L, 128], every frequency repeated twice."""
    cos_out, sin_out = [], []
    pos = ids.float()
    for i, d in enumerate(axes_dim):
        freqs = 1.0 / (theta ** (torch.arange(0, d, 2, dtype=torch.float64, device=ids.device)[: d // 2] / d))
        ang = torch.outer(pos[:, i].double(), freqs)
        cos_out.append(ang.cos().repeat_interleave(2, dim=1).float())
        sin_out.append(ang.sin().repeat_interleave(2, dim=1).float())
    return torch.cat(cos_out, dim=-1).contiguous(), torch.cat(sin_out, dim=-1).contiguous()


class _MLPEmbedder(nn.Module):
    """TimestepEmbedding / PixArtAlphaTextProjection: linear_1 -> SiLU -> linear_2."""

    def __init__(self, in_dim, dim, dtype, device):
        super().__init__()
        self.linear_1 = _plain(dim, in_dim, dtype, device)
        self.linear_2 = _plain(dim, dim, dtype, device)

    def forward(self, x):
        h = linear(x, self.linear_1)
        h = torch.nn.functional.silu(h.float()).to(torch.bfloat16)
        return linear(h, self.linear_2)


class CombinedTimestepGuidanceTextProjEmbeddings(nn.Module):
    def __init__(self, dim, pooled_dim, dtype, device, guidance=True):
        super().__init__()
        self.timestep_embedder = _MLPEmbedder(256, dim, dtype, device)
        if guidance:
            self.guidance_embedder = _MLPEmbedder(256, dim, dtype, device)
        self.text_embedder = _MLPEmbedder(pooled_dim, dim, dtype, device)

    def forward(self, timestep, guidance, pooled):
        emb = self.timestep_embedder(timestep_sinusoid(timestep).to(torch.bfloat16))
        if guidance is not None and hasattr(self, 'guidance_embedder') and not getattr(self, 'bypass_guidance', False):
            emb = emb + self.guidance_embedder(timestep_sinusoid(guidance).to(torch.bfloat16))
        return emb + self.text_embedder(pooled)


class FluxTransformer2DModel(nn.Module):
    """Parameter tree with diffusers' names (x_embedder, time_text_embed, context_embedder, transformer_blocks,
    single_transformer_blocks, norm_out, proj_out)."""

    def __init__(self, cfg=None, dtype=torch.bfloat16, device='cuda'):
        super().__init__()
        cfg = dict(FLUX_DEV_CONFIG, **(cfg or {}))
        self.config = cfg
        heads, hd = cfg['num_attention_heads'], cfg['attention_head_dim']
        assert hd == 128, 'kernels are specialised for head_dim 128'
        dim = heads * hd
        self.inner_dim = dim
        self.axes_dim = tuple(cfg['axes_dims_rope'])
        self.x_embedder = _plain(dim, cfg['in_channels'], dtype, device)
        self.time_text_embed = CombinedTimestepGuidanceTextProjEmbeddings(dim, cfg['pooled_projection_dim'], dtype, device,
                                                                          cfg.get('guidance_embeds', True))
        self.context_embedder = _plain(dim, cfg['joint_attention_dim'], dtype, device)
        self.transformer_blocks = nn.ModuleList(
            [FluxTransformerBlock(dim, heads, 4, dtype, device) for _ in range(cfg['num_layers'])])
        self.single_transformer_blocks = nn.ModuleList(
            [FluxSingleTransformerBlock(dim, heads, 4, dtype, device) for _ in range(cfg['num_single_layers'])])
        self.norm_out = _AdaNorm(dim, 2, dtype, device)
        self.proj_out = _plain(cfg['in_channels'], dim, dtype, device)
        for name, p in self.named_parameters():
            p.original_name = name   # models/flux.py:212-213


def make_contiguous(*values):
    return tuple(x.contiguous() if torch.is_tensor(x) else x for x in values)


# =====================================================================================================================
# pipeline layers (models/flux.py:456-548)
# =====================================================================================================================
class EmbeddingWrapper(nn.Module):
    def __init__(self, x_embedder, time_text_embed, context_embedder, axes_dim):
        super().__init__()
        self.x_embedder = x_embedder
        self.time_text_embed = time_text_embed
        self.context_embedder = context_embedder
        self.axes_dim = axes_dim

    def forward(self, inputs):
        for item in inputs:
            if torch.is_floating_point(item):
                item.requires_grad_(True)
        hidden_states, encoder_hidden_states, pooled_projections, timestep, img_ids, txt_ids, guidance, img_seq_len = inputs
        hidden_states = linear(hidden_states, self.x_embedder)
        timestep = timestep.to(torch.bfloat16) * 1000
        guidance = guidance.to(torch.bfloat16) * 1000
        has_g = hasattr(self.time_text_embed, 'guidance_embedder')
        temb = self.time_text_embed(timestep, guidance if has_g else None, pooled_projections.to(torch.bfloat16))
        encoder_hidden_states = linear(encoder_hidden_states, self.context_embedder)
        if txt_ids.ndim == 3:
            txt_ids = txt_ids[0]
        if img_ids.ndim == 3:
            img_ids = img_ids[0]
        freqs_cos, freqs_sin = flux_rope_tables(torch.cat((txt_ids, img_ids), dim=0), self.axes_dim)
        return make_contiguous(hidden_states, encoder_hidden_states, temb, freqs_cos, freqs_sin, img_seq_len)


class TransformerWrapper(nn.Module):
    def __init__(self, block, block_idx):
        super().__init__()
        self.block = block
        self.block_idx = block_idx

    def forward(self, inputs):
        hidden_states, encoder_hidden_states, temb, freqs_cos, freqs_sin, img_seq_len = inputs
        encoder_hidden_states, hidden_states = self.block(
            hidden_states=hidden_states, encoder_hidden_states=encoder_hidden_states, temb=temb,
            image_rotary_emb=(freqs_cos, freqs_sin))
        return make_contiguous(hidden_states, encoder_hidden_states, temb, freqs_cos, freqs_sin, img_seq_len)


class SingleTransformerWrapper(TransformerWrapper):
    pass


class OutputWrapper(nn.Module):
    def __init__(self, norm_out, proj_out):
        super().__init__()
        self.norm_out = norm_out
        self.proj_out = proj_out

    def forward(self, inputs):
        hidden_states, encoder_hidden_states, temb, freqs_cos, freqs_sin, img_seq_len = inputs
        # The reference slices `hidden_states[:, :img_seq_len[0].item()]` here (models/flux.py:545-546) — a host sync per
        # micro-batch whose only effect is to drop Kontext control tokens.  The prediction is computed for every token
        # instead and the loss keeps the first target.shape[1] of them (shape metadata, no device read).
        hidden_states = AdaLNContinuousFn.apply(hidden_states, temb, self.norm_out.linear)
        return linear(hidden_states, self.proj_out)


# =====================================================================================================================
# the plugin
# =====================================================================================================================
def time_shift(mu, sigma, t):
    return math.exp(mu) / (math.exp(mu) + (1 / t - 1) ** sigma)


def get_lin_function(x1=256, y1=0.5, x2=4096, y2=1.15):
    m = (y2 - y1) / (x2 - x1)
    b = y1 - m * x1
    return lambda x: m * x + b


def pack_latents(x):
    """'b c (h ph) (w pw) -> b (h w) (c ph pw)' with ph = pw = 2 (models/flux.py:377-378)."""
    b, c, h, w = x.shape
    return x.view(b, c, h // 2, 2, w // 2, 2).permute(0, 2, 4, 1, 3, 5).reshape(b, (h // 2) * (w // 2), c * 4)


def latent_image_ids(h2, w2, device=None, dtype=torch.float32):
    ids = torch.zeros(h2, w2, 3, device=device, dtype=dtype)
    ids[..., 1] = ids[..., 1] + torch.arange(h2, device=device)[:, None]
    ids[..., 2] = ids[..., 2] + torch.arange(w2, device=device)[None, :]
    return ids.reshape(h2 * w2, 3)


def base_storage_dtype(model_config, adapter_configured=True):
    """`transformer_dtype` of the reference (models/flux.py:172,203-205; utils/common.py:18-20): None when the frozen base
    stays in the compute dtype, torch.float8_e4m3fn / float8_e5m2 when the 2-D weights of the blocks are stored in fp8 and
    widened by csrc/fp8_dequant.cu in front of every GEMM that reads them (LoRA runs only: an fp8 base cannot be trained)"""
    v = model_config.get('transformer_dtype', None)
    if isinstance(v, str):
        v = {'bfloat16': torch.bfloat16, 'float8': torch.float8_e4m3fn, 'float8_e4m3fn': torch.float8_e4m3fn,
             'float8_e5m2': torch.float8_e5m2}.get(v, v)
    if v is None or v == torch.bfloat16:
        return None
    if v not in (torch.float8_e4m3fn, torch.float8_e5m2):
        raise NotImplementedError(f'transformer_dtype {v!r}: bfloat16, float8 (e4m3fn) and float8_e5m2 are supported')
    if not adapter_configured:
        raise NotImplementedError('transformer_dtype float8 needs an [adapter]: a float8 base is frozen storage, not trainable')
    return v


class FluxPipeline(PluginSurface):
    """Mirror of the reference FluxPipeline's training-side surface (models/flux.py:153-404)."""
    name = 'flux'
    checkpointable_layers = ['TransformerWrapper', 'SingleTransformerWrapper']
    adapter_target_modules = ['FluxTransformerBlock', 'FluxSingleTransformerBlock']
    framerate = None
    pixels_round_to_multiple = 16

    def __init__(self, config, device='cuda'):
        self.config = config
        self.model_config = config['model']
        dtype = self.model_config.get('dtype', torch.bfloat16)
        if isinstance(dtype, str):
            dtype = {'bfloat16': torch.bfloat16, 'float16': torch.float16, 'float32': torch.float32}[dtype]
        if dtype != torch.bfloat16:
            raise NotImplementedError('the sm_90a Flux path computes in bf16 (model.dtype must be bfloat16)')
        tcfg = self.model_config.get('transformer_config', None)
        # models/flux.py:174-191: without `transformer_path` the weights are `<diffusers_path>/transformer/*.safetensors`,
        # whose config.json describes the architecture (dev / schnell)
        dpath = self.model_config.get('diffusers_path', None)
        if dpath and not self.model_config.get('transformer_path', None) and os.path.isdir(os.path.join(dpath, 'transformer')):
            self.model_config['transformer_path'] = os.path.join(dpath, 'transformer')
            cfg_json = os.path.join(dpath, 'transformer', 'config.json')
            if tcfg is None and os.path.exists(cfg_json):
                tcfg = cfg_json
        if isinstance(tcfg, str):
            with open(tcfg) as f:
                tcfg = {k: v for k, v in json.load(f).items() if k in FLUX_DEV_CONFIG}
        self.tcfg = dict(FLUX_DEV_CONFIG, **(tcfg or {}))
        device = self.model_config.get("device", device)      # (tests: "cpu" with the kernel test doubles)
        self.dtype, self.device = dtype, device
        self.pipeline_model = None
        self.model_engine = None
        self.adapter_config = None
        if self.model_config.get('lazy_layers', False):
            # Stage-local construction: to_layers() hands the engine LayerSpecs and only the layers of this rank's
            # stage are ever materialised (12 B parameters do not fit eight times on the host, and need not).
            self.transformer = None
            return
        self.transformer = FluxTransformer2DModel(self.tcfg, dtype=dtype, device=device)
        if path := self.model_config.get('transformer_path', None):
            self.load_transformer_weights(path)
        if self.model_config.get('bypass_guidance_embedding', False):       # models/flux.py:132-150,191-194
            self.transformer.time_text_embed.bypass_guidance = True
        self.transformer.train()

    def _lazy_layers(self):
        from .pipe.module import LayerSpec
        cfg, dtype, device = self.tcfg, self.dtype, self.device
        heads = cfg['num_attention_heads']
        dim = heads * cfg['attention_head_dim']

        def name_params(module, prefix_map):
            for n, p in module.named_parameters():
                for local, glob in prefix_map.items():
                    if n.startswith(local):
                        p.original_name = glob + n[len(local):]
                        break
            return module

        def build_embed(dev=None):
            d = dev or device
            w = EmbeddingWrapper(_plain(dim, cfg['in_channels'], dtype, d),
                                 CombinedTimestepGuidanceTextProjEmbeddings(dim, cfg['pooled_projection_dim'], dtype, d,
                                                                            cfg.get('guidance_embeds', True)),
                                 _plain(dim, cfg['joint_attention_dim'], dtype, d), tuple(cfg['axes_dims_rope']))
            if self.model_config.get('bypass_guidance_embedding', False):
                w.time_text_embed.bypass_guidance = True
            return self._adapt(name_params(w, {'x_embedder.': 'x_embedder.', 'time_text_embed.': 'time_text_embed.',
                                               'context_embedder.': 'context_embedder.'}), dev)

        def build_double(i, dev=None):
            w = TransformerWrapper(FluxTransformerBlock(dim, heads, 4, dtype, dev or device), i)
            return self._adapt(name_params(w, {'block.': f'transformer_blocks.{i}.'}), dev)

        def build_single(i, dev=None):
            w = SingleTransformerWrapper(FluxSingleTransformerBlock(dim, heads, 4, dtype, dev or device), i)
            return self._adapt(name_params(w, {'block.': f'single_transformer_blocks.{i}.'}), dev)

        def build_out(dev=None):
            d = dev or device
            w = OutputWrapper(_AdaNorm(dim, 2, dtype, d), _plain(cfg['in_channels'], dim, dtype, d))
            return self._adapt(name_params(w, {'norm_out.': 'norm_out.', 'proj_out.': 'proj_out.'}), dev)

        def count(fn, *a):
            return sum(p.numel() for p in fn(*a, dev='meta').parameters())

        def spec(cls, fn, *a, n):
            s = LayerSpec(cls, *a)
            s.build = lambda fn=fn, a=a: fn(*a)
            s.param_count = n
            return s
        n_double, n_single = count(build_double, 0), count(build_single, 0)
        layers = [spec(EmbeddingWrapper, build_embed, n=count(build_embed))]
        layers += [spec(TransformerWrapper, build_double, i, n=n_double) for i in range(cfg['num_layers'])]
        layers += [spec(SingleTransformerWrapper, build_single, i, n=n_single) for i in range(cfg['num_single_layers'])]
        layers.append(spec(OutputWrapper, build_out, n=count(build_out)))
        return layers

    # ---- weights ----
    @staticmethod
    def _weight_index(path):
        """{parameter name: (file, key in file)} over a *.safetensors file or a directory of shards (diffusers / reference
        parameter names; ComfyUI checkpoints carry `model.diffusion_model.` in front, models/wan/wan.py:43-46).  Only the
        headers are read here; tensors are fetched one by one when a layer asks for them."""
        from safetensors import safe_open
        files = [path] if os.path.isfile(path) else sorted(
            os.path.join(path, f) for f in os.listdir(path) if f.endswith('.safetensors'))
        if not files:
            raise RuntimeError(f'no *.safetensors under {path}')
        index = {}
        for f in files:
            with safe_open(f, framework='pt') as h:
                for k in h.keys():
                    index[re.sub(r'^model\.diffusion_model\.', '', k)] = (f, k)
        return index

    @staticmethod
    def _copy_weights(index, named_params, what):
        """fills every (name, parameter) from the checkpoint; a parameter the checkpoint does not have raises"""
        from safetensors import safe_open
        named_params = list(named_params)
        if 'img_in.weight' in index and 'x_embedder.weight' not in index:
            return FluxPipeline._copy_bfl_weights(index, named_params, what)
        by_file, missing = {}, []
        for name, p in named_params:
            if name in index:
                by_file.setdefault(index[name][0], []).append((index[name][1], name, p))
            else:
                missing.append(name)
        if missing:
            raise RuntimeError(f'{len(missing)} parameters of {what} missing from the checkpoint, e.g. {sorted(missing)[:3]}')
        with torch.no_grad():
            for f, items in by_file.items():
                with safe_open(f, framework='pt') as h:
                    for key, name, p in items:
                        v = h.get_tensor(key)
                        if tuple(v.shape) != tuple(p.shape):
                            raise RuntimeError(f'{name}: checkpoint shape {tuple(v.shape)} != parameter shape {tuple(p.shape)}')
                        p.copy_(v)

    @staticmethod
    def _copy_bfl_weights(index, named_params, what):
        """the checkpoint is in the BFL / ComfyUI layout (img_in, double_blocks.N.img_attn.qkv, ...): every parameter is a
        row range of a BFL tensor (flux_export.from_bfl_plan)"""
        from safetensors import safe_open
        from .flux_export import from_bfl_plan, read_bfl_tensor
        plan = from_bfl_plan([(n, tuple(p.shape)) for n, p in named_params])
        missing = sorted(n for n, (bk, _, _, _) in plan.items() if bk not in index)
        if missing:
            raise RuntimeError(f'{len(missing)} parameters of {what} missing from the checkpoint, e.g. {missing[:3]}')
        with torch.no_grad():
            for name, p in named_params:
                bk, off, rows, swap = plan[name]
                f, key = index[bk]
                with safe_open(f, framework='pt') as h:
                    v = read_bfl_tensor(h.get_tensor(key), off, rows, swap)
                if tuple(v.shape) != tuple(p.shape):
                    raise RuntimeError(f'{name}: checkpoint shape {tuple(v.shape)} != parameter shape {tuple(p.shape)}')
                p.copy_(v)

    def load_transformer_weights(self, path):
        """Loads a checkpoint in the reference's parameter names into the whole (eagerly built) transformer."""
        FluxPipeline._copy_weights(FluxPipeline._weight_index(path), list(self.transformer.named_parameters()), 'the transformer')

    def _load_stage_weights(self, module):
        """lazily built layers (`lazy_layers`): each rank reads exactly the tensors of the layers it materialises, by
        `original_name` — nothing when no `transformer_path` is configured (synthetic / benchmark runs)"""
        path = self.model_config.get('transformer_path', None)
        if not path:
            return
        if getattr(self, '_windex', None) is None:
            self._windex = FluxPipeline._weight_index(path)
        FluxPipeline._copy_weights(self._windex, [(getattr(p, 'original_name', n), p) for n, p in module.named_parameters()],
                                   type(module).__name__)

    def load_diffusion_model(self):
        pass

    # ---- adapters (models/base.py:263-303, train.py:531-535) ----
    def configure_adapter(self, adapter_config):
        """LoRA on every Linear of the transformer blocks, everything else frozen (lora.py).  Call before to_layers() /
        the engine is built, as the reference does (train.py:531 precedes :597)."""
        if adapter_config.get('type', 'lora') != 'lora':
            raise NotImplementedError(f"adapter type {adapter_config.get('type')!r}: only 'lora' is built for the sm_90a path")
        if adapter_config.get('dropout', 0.0):
            raise NotImplementedError('lora dropout > 0 is not supported on the sm_90a path')
        self.adapter_config = dict(adapter_config)
        if self.transformer is not None:
            self._adapt(self.transformer, None)

    def _adapt(self, module, dev):
        """freezes `module` and attaches the configured adapters to the blocks inside it (no-op without an adapter or on
        the meta device used for parameter counting)"""
        if dev == 'meta':
            return module
        if self.transformer is None:                       # lazy_layers: this is where a stage-local layer gets its weights
            FluxPipeline._load_stage_weights(self, module)
        if self.adapter_config is None:
            return module
        from . import lora
        for p in module.parameters():
            p.requires_grad_(False)
        dtype = self.adapter_config.get('dtype', torch.bfloat16)
        if isinstance(dtype, str):
            dtype = {'bfloat16': torch.bfloat16, 'float32': torch.float32}[dtype]
        if dtype != torch.bfloat16:
            raise NotImplementedError('adapter dtype must be bfloat16 on the sm_90a path')
        lora.attach(module, int(self.adapter_config['rank']), dtype, base_storage_dtype(self.model_config))
        if getattr(self, '_adapter_init', None) is not None:
            FluxPipeline._load_factors(module, self._adapter_init)
        return module

    def load_adapter_weights(self, adapter_path):
        """models/base.py:367-388 (train.py:534-535, `[adapter] init_from_existing`): start the factors from a saved
        adapter — the single *.safetensors file in `adapter_path`, keys optionally prefixed `transformer.` /
        `diffusion_model.`; a key that names no parameter of the model raises.  With lazily built layers the file is
        read once and every stage fills the blocks it builds."""
        from safetensors.torch import load_file
        files = sorted(f for f in os.listdir(adapter_path) if f.endswith('.safetensors'))
        if len(files) == 0:
            raise RuntimeError(f'No safetensors file found in {adapter_path}')
        if len(files) > 1:
            raise RuntimeError(f'Multiple safetensors files found in {adapter_path}')
        state = {re.sub(r'^(transformer|diffusion_model)\.', '', k): v
                 for k, v in load_file(os.path.join(adapter_path, files[0])).items()}
        self._adapter_init = state
        if self.transformer is not None:
            names = {n for n, _ in self.transformer.named_parameters()}
            for k in state:
                if k not in names:
                    raise RuntimeError(f'adapter key {k} is not in the model parameters')
            FluxPipeline._load_factors(self.transformer, state)

    @staticmethod
    def _load_factors(module, state):
        with torch.no_grad():
            for n, p in module.named_parameters():
                if '.lora_A.' in n or '.lora_B.' in n:
                    key = getattr(p, 'original_name', n)
                    if key in state:
                        if tuple(state[key].shape) != tuple(p.shape):
                            raise RuntimeError(f'adapter key {key}: shape {tuple(state[key].shape)} does not match {tuple(p.shape)}')
                        p.copy_(state[key].to(p.dtype))

    def save_model(self, save_dir, state_dict):
        """full-model export: the BFL / ComfyUI layout the reference writes (models/flux.py:257-288; flux_export.py), or the
        diffusers names this engine trains in with `[model] export_layout = 'diffusers'`"""
        if self.model_config.get('export_layout', 'bfl') == 'bfl':
            from .flux_export import to_bfl
            state_dict = to_bfl(state_dict)
        FluxPipeline.write_model_file(save_dir, state_dict)

    @staticmethod
    def write_model_file(save_dir, state_dict):
        from safetensors.torch import save_file
        os.makedirs(save_dir, exist_ok=True)
        save_file({k: v.contiguous() for k, v in state_dict.items()}, os.path.join(save_dir, 'model.safetensors'),
                  metadata={'format': 'pt'})

    def save_adapter(self, save_dir, peft_state_dict):
        """models/flux.py:231-236: diffusers' `save_lora_weights(save_dir, transformer_lora_layers=...)` — one file
        `pytorch_lora_weights.safetensors` whose keys carry the `transformer.` component prefix (diffusers' convention,
        recalled: diffusers is absent); load_adapter_weights strips it again"""
        FluxPipeline.write_adapter_file(save_dir, {'transformer.' + k: v for k, v in peft_state_dict.items()},
                                        'pytorch_lora_weights.safetensors')

    @staticmethod
    def write_adapter_file(save_dir, state_dict, filename='adapter_model.safetensors'):
        from safetensors.torch import save_file
        os.makedirs(save_dir, exist_ok=True)
        save_file({k: v.contiguous() for k, v in state_dict.items()}, os.path.join(save_dir, filename), metadata={'format': 'pt'})

    def write_peft_config(self, save_dir, peft_state_dict):
        """`peft_config.save_pretrained(save_dir)` of the Qwen-Image / Wan exports (models/qwen_image.py:291,
        models/wan/wan.py:259): adapter_config.json with the fields of the LoraConfig the reference builds
        (models/base.py:272-303: r, lora_alpha = r, dropout, bias 'none', the adapted Linear modules)"""
        ac = self.adapter_config or {}
        mods = sorted({re.sub(r'\.lora_[AB]\.weight$', '', k) for k in peft_state_dict})
        cfg = {'peft_type': 'LORA', 'r': int(ac.get('rank', 0)), 'lora_alpha': int(ac.get('alpha', ac.get('rank', 0))),
               'lora_dropout': float(ac.get('dropout', 0.0)), 'bias': 'none', 'target_modules': mods, 'inference_mode': True,
               'base_model_name_or_path': None, 'task_type': None}
        os.makedirs(save_dir, exist_ok=True)
        with open(os.path.join(save_dir, 'adapter_config.json'), 'w') as f:
            json.dump(cfg, f, indent=2)

    def get_param_groups(self, parameters):
        return [{'params': parameters}]

    def model_specific_dataset_config_validation(self, dataset_config):
        pass

    # ---- data -> model inputs (models/flux.py:323-394) ----
    def prepare_inputs(self, inputs, timestep_quantile=None):
        latents = inputs['latents'].float()
        clip_embed = inputs['clip_embed']
        t5_embed = inputs['t5_embed']
        mask = inputs['mask']
        bs, c, h, w = latents.shape
        if mask is not None:
            mask = mask.unsqueeze(1).expand((-1, c, -1, -1))
            mask = torch.nn.functional.interpolate(mask, size=(h, w), mode='nearest-exact')
            mask = pack_latents(mask)
        img_ids = latent_image_ids(h // 2, w // 2, latents.device, latents.dtype).unsqueeze(0).repeat((bs, 1, 1))
        txt_ids = torch.zeros(bs, t5_embed.shape[1], 3).to(latents.device, latents.dtype)
        method = self.model_config.get('timestep_sample_method', 'logit_normal')
        if method == 'logit_normal':
            dist = torch.distributions.normal.Normal(0, 1)
        elif method == 'uniform':
            dist = torch.distributions.uniform.Uniform(0, 1)
        else:
            raise NotImplementedError()
        if timestep_quantile is not None:
            t = dist.icdf(torch.full((bs,), timestep_quantile, device=latents.device))
        else:
            t = dist.sample((bs,)).to(latents.device)
        if method == 'logit_normal':
            t = torch.sigmoid(t * self.model_config.get('sigmoid_scale', 1.0))
        if shift := self.model_config.get('shift', None):
            t = (t * shift) / (1 + (shift - 1) * t)
        elif self.model_config.get('flux_shift', False):
            mu = get_lin_function(y1=0.5, y2=1.15)((h // 2) * (w // 2))
            t = time_shift(mu, 1.0, t)
        x_1 = latents
        x_0 = torch.randn_like(x_1)
        if self._noise_on_device(x_1):
            # SURVEY 8(f)4: t and x_0 come from the host RNG in the reference's order; mix + target + packing run on the device
            x_t, target = ops.noise_on_device(x_1, x_0, t, True, self.device)
            guidance_vec = torch.full((bs,), float(self.model_config.get('guidance', 1.0)), dtype=torch.float32)
        else:
            te = t.view(-1, 1, 1, 1)
            x_t = (1 - te) * x_1 + te * x_0
            target = x_0 - x_1
            guidance_vec = torch.full((bs,), float(self.model_config.get('guidance', 1.0)), device=x_t.device,
                                      dtype=torch.float32)
            x_t = pack_latents(x_t)
            target = pack_latents(target)
        img_seq_len = torch.tensor(x_t.shape[1], device=latents.device).repeat((bs,))
        if 'control_latents' in inputs:
            control = inputs['control_latents'].float().to(x_t.device)
            assert control.shape == latents.shape
            cids = latent_image_ids(h // 2, w // 2, control.device, control.dtype)
            cids[..., 0] = 1
            img_ids = torch.cat([img_ids, cids.unsqueeze(0).repeat((bs, 1, 1))], dim=1)
            x_t = torch.cat([x_t, pack_latents(control)], dim=1)
        return (x_t, t5_embed, clip_embed, t, img_ids, txt_ids, guidance_vec, img_seq_len), (target, mask)

    # ---- layers / loss ----
    def to_layers(self):
        base_storage_dtype(self.model_config, self.adapter_config is not None)
        if self.transformer is None:
            return self._lazy_layers()
        t = self.transformer
        layers = [EmbeddingWrapper(t.x_embedder, t.time_text_embed, t.context_embedder, t.axes_dim)]
        for i, block in enumerate(t.transformer_blocks):
            layers.append(TransformerWrapper(block, i))
        for i, block in enumerate(t.single_transformer_blocks):
            layers.append(SingleTransformerWrapper(block, i))
        layers.append(OutputWrapper(t.norm_out, t.proj_out))
        return layers

    def get_loss_fn(self):
        cfg = self.config

        def loss_fn(output, label):
            target, mask = label
            if 'huber_delta' in cfg or 'smooth_l1_beta' in cfg:
                # non-default robust losses are not on the benchmarked hot path: ATen elementwise on the device
                o, t = output.float(), target.to(output.device, torch.float32)
                if 'huber_delta' in cfg:
                    loss = torch.nn.functional.huber_loss(o, t, reduction='none', delta=cfg['huber_delta'])
                else:
                    loss = torch.nn.functional.smooth_l1_loss(o, t, reduction='none', beta=cfg['smooth_l1_beta'])
                if mask.numel() > 0:
                    loss = loss * mask.to(o.device, torch.float32)
                return loss.mean()
            if output.shape[1] != target.shape[1]:
                output = output[:, :target.shape[1]]
            m = mask.to(output.device) if mask.numel() > 0 else None
            return MseLossFn.apply(output, target.to(output.device), m)
        return loss_fn
