"""Qwen-Image on the sm_90a kernels — the drop-in for the reference's models/qwen_image.py (SURVEY.md row Q1).

Same plugin surface as the reference's QwenImagePipeline (models/qwen_image.py:177-517): `name`,
`checkpointable_layers`, `prepare_inputs(batch, timestep_quantile)`, `to_layers()`, `get_loss_fn()`, and layers that
speak its tuple protocol `(hidden_states, encoder_hidden_states, attention_mask, temb, vid_freqs, txt_freqs, *extra)`
(models/qwen_image.py:519-605).

The Qwen-Image block (diffusers QwenImageTransformerBlock driven by the reference's QwenDoubleStreamAttnProcessor2_0,
models/qwen_image.py:91-174) is arithmetically the Flux double-stream block: AdaLN-zero modulation with chunk order
(shift, scale, gate) x (attention, mlp), biased q/k/v projections, per-head RMSNorm(1e-6) on q and k, interleaved-pair
RoPE in fp32, joint attention over [text, image], gated residuals, GELU(tanh) MLP.  It therefore runs on
`FluxDoubleBlockFn` (flux_blocks.py) unchanged; this file supplies the parameter tree under diffusers' Qwen names
(img_mod.1, txt_mod.1, attn.*, img_mlp, txt_mlp), the embedders, the rope tables of diffusers'
QwenEmbedRope(scale_rope=True) and the pipeline layers.

Two deliberate differences from the reference's tuple contents (both internal to these layers):
  * vid_freqs / txt_freqs travel as real fp32 `[2, tokens, 128]` (cos, sin; every frequency repeated twice) instead
    of complex64 `[tokens, 64]`: the same numbers in the form the fused q/k-norm+RoPE epilogue consumes;
  * the bool key mask (models/qwen_image.py:472-476) is not carried into the attention kernel as a mask.  prepare_inputs
    pads every prompt of a step's batch (micro-batch x GAS examples) to the longest one, so padded prompts are the normal
    case with real captions; InitialLayer always appends the real lengths to the tuple (one int32 tensor, last element —
    always, so that every micro-batch of a step has the same tuple structure on the stage links) and, when any prompt
    is shorter than the padded length, every block attends per sample over its valid rows
    (flux_blocks._ragged_attn_fwd): same loss and gradients as masking, on the same dense kernels.  Micro-batches whose
    prompts all fill the padded length take the unmasked path.  Masks with holes inside a prompt raise
    NotImplementedError.
"""
import json
import math

import torch
from torch import nn

from . import ops
from .flux import AdaLNContinuousFn, MseLossFn, _MLPEmbedder, get_lin_function, linear, make_contiguous, time_shift
from .flux_blocks import HD, FluxDoubleBlockFn, FusedParam, _AdaNorm, _Attn, _FF, _norm_w, _plain, double_block_sites
from .plugin import PluginSurface

QWEN_IMAGE_CONFIG = {   # reference: configs/qwen_image/transformer/config.json
    'attention_head_dim': 128, 'num_attention_heads': 24, 'num_layers': 60, 'in_channels': 64, 'out_channels': 16,
    'joint_attention_dim': 3584, 'patch_size': 2, 'axes_dims_rope': [16, 56, 56], 'guidance_embeds': False,
}


class _Alias:
    """attribute bag that is NOT an nn.Module (so aliased parameters are not registered twice)"""

    def __init__(self, **kw):
        self.__dict__.update(kw)


class QwenImageTransformerBlock(nn.Module):
    """Drop-in for diffusers' QwenImageTransformerBlock (same parameter names; call signature as used at
    models/qwen_image.py:570-577); returns (encoder_hidden_states, hidden_states)."""

    def __init__(self, dim=3072, heads=24, mlp_ratio=4, dtype=torch.bfloat16, device='cuda'):
        super().__init__()
        assert dim == heads * HD
        self.dim, self.heads = dim, heads
        self.img_mod = nn.Sequential(nn.SiLU(), _plain(6 * dim, dim, dtype, device))
        self.txt_mod = nn.Sequential(nn.SiLU(), _plain(6 * dim, dim, dtype, device))
        qkv = FusedParam([dim] * 3, dim, dtype, device)
        add_qkv = FusedParam([dim] * 3, dim, dtype, device)
        a = _Attn()
        a.to_q, a.to_k, a.to_v = qkv.lin(0), qkv.lin(1), qkv.lin(2)
        a.add_q_proj, a.add_k_proj, a.add_v_proj = add_qkv.lin(0), add_qkv.lin(1), add_qkv.lin(2)
        a.norm_q, a.norm_k = _norm_w(dtype, device), _norm_w(dtype, device)
        a.norm_added_q, a.norm_added_k = _norm_w(dtype, device), _norm_w(dtype, device)
        a.to_out = nn.ModuleList([_plain(dim, dim, dtype, device), nn.Identity()])
        a.to_add_out = _plain(dim, dim, dtype, device)
        self.attn = a
        self.img_mlp = _FF(dim, dim * mlp_ratio, dtype, device)
        self.txt_mlp = _FF(dim, dim * mlp_ratio, dtype, device)
        # the Flux names lora.attach_double_block reads (plain attributes: no second registration of the same parameters)
        d = self.__dict__
        d['qkv'], d['add_qkv'] = qkv, add_qkv
        d['norm1'] = _Alias(linear=self.img_mod[1])
        d['norm1_context'] = _Alias(linear=self.txt_mod[1])
        d['ff'], d['ff_context'] = self.img_mlp, self.txt_mlp
        self.sites = double_block_sites(self.img_mod[1], self.txt_mod[1], qkv, add_qkv, a, self.img_mlp, self.txt_mlp)

    def forward(self, hidden_states, encoder_hidden_states, temb, image_rotary_emb, encoder_hidden_states_mask=None,
                joint_attention_kwargs=None, txt_lens=None):
        """txt_lens: None, or the real prompt length of every sample when the micro-batch is padded (key mask)"""
        cos, sin = image_rotary_emb            # joint [text; image] tables, fp32 [L, 128]
        h, e = FluxDoubleBlockFn.apply(self, hidden_states, encoder_hidden_states, temb, cos, sin, txt_lens)
        return e, h


def qwen_rope_tables(img_shapes, txt_len, axes_dim=(16, 56, 56), theta=10000.0, device=None):
    """diffusers QwenEmbedRope(theta=10000, axes_dim, scale_rope=True): image tokens of entry idx = (frame, h, w) sit at
    (idx + f, y - (h - h//2), x - (w - w//2)); text tokens at max(h//2, w//2) + i on all three axes
    (models/qwen_image.py:537-538 calls it; rope_params :547-555).  Returns (vid [2, Li, 128], txt [2, Lt, 128]) fp32:
    cos and sin with every frequency repeated twice (the real form of the complex freqs_cis of :66-71)."""
    def angles(pos, d):
        freqs = 1.0 / torch.pow(torch.tensor(theta, dtype=torch.float32, device=device),
                                torch.arange(0, d, 2, device=device).to(torch.float32).div(d))
        return torch.outer(pos.to(torch.float32), freqs)

    vid, max_idx = [], 0
    for idx, (frame, h, w) in enumerate(img_shapes):
        pf = torch.arange(idx, idx + frame, device=device)
        ph = torch.arange(h, device=device) - (h - h // 2)
        pw = torch.arange(w, device=device) - (w - w // 2)
        a = torch.cat([angles(pf, axes_dim[0]).view(frame, 1, 1, -1).expand(frame, h, w, -1),
                       angles(ph, axes_dim[1]).view(1, h, 1, -1).expand(frame, h, w, -1),
                       angles(pw, axes_dim[2]).view(1, 1, w, -1).expand(frame, h, w, -1)], dim=-1)
        vid.append(a.reshape(frame * h * w, -1))
        max_idx = max(max_idx, h // 2, w // 2)
    vid = torch.cat(vid, dim=0)
    txt = torch.cat([angles(torch.arange(max_idx, max_idx + txt_len, device=device), d) for d in axes_dim], dim=-1)

    def pair(a):
        return torch.stack([a.cos().repeat_interleave(2, dim=1), a.sin().repeat_interleave(2, dim=1)]).contiguous()
    return pair(vid), pair(txt)


class QwenTimestepProjEmbeddings(nn.Module):
    """diffusers QwenTimestepProjEmbeddings: Timesteps(256, flip_sin_to_cos=True, downscale_freq_shift=0, scale=1000)
    followed by TimestepEmbedding(256, dim); the pooled projection of Flux does not exist here."""

    def __init__(self, dim, dtype, device):
        super().__init__()
        self.timestep_embedder = _MLPEmbedder(256, dim, dtype, device)

    def forward(self, timestep):
        half = 128
        exponent = -math.log(10000.0) * torch.arange(0, half, dtype=torch.float32, device=timestep.device) / half
        emb = 1000.0 * (timestep[:, None].float() * torch.exp(exponent)[None, :])
        proj = torch.cat([torch.cos(emb), torch.sin(emb)], dim=-1)
        return self.timestep_embedder(proj.to(torch.bfloat16))


class _RMSNormW(nn.Module):
    """diffusers RMSNorm(dim, eps=1e-6) with scale: fp32 statistics, bf16 result (txt_norm; [Lt, 3584] once per
    micro-batch — ATen elementwise, not a hot-path kernel)."""

    def __init__(self, dim, dtype, device, eps=1e-6):
        super().__init__()
        self.eps = eps
        self.weight = nn.Parameter(torch.ones(dim, dtype=dtype, device=device))

    def forward(self, x):
        xf = x.float()
        xh = (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + self.eps)).to(self.weight.dtype)
        return xh * self.weight


class QwenImageTransformer2DModel(nn.Module):
    """Parameter tree with diffusers' names (img_in, txt_norm, txt_in, time_text_embed, transformer_blocks, norm_out,
    proj_out)."""

    def __init__(self, cfg=None, dtype=torch.bfloat16, device='cuda'):
        super().__init__()
        cfg = dict(QWEN_IMAGE_CONFIG, **(cfg or {}))
        self.config = cfg
        heads, hd = cfg['num_attention_heads'], cfg['attention_head_dim']
        assert hd == HD, 'kernels are specialised for head_dim 128'
        dim = heads * hd
        self.inner_dim = dim
        self.axes_dim = tuple(cfg['axes_dims_rope'])
        self.img_in = _plain(dim, cfg['in_channels'], dtype, device)
        self.txt_norm = _RMSNormW(cfg['joint_attention_dim'], dtype, device)
        self.txt_in = _plain(dim, cfg['joint_attention_dim'], dtype, device)
        self.time_text_embed = QwenTimestepProjEmbeddings(dim, dtype, device)
        self.transformer_blocks = nn.ModuleList(
            [QwenImageTransformerBlock(dim, heads, 4, dtype, device) for _ in range(cfg['num_layers'])])
        self.norm_out = _AdaNorm(dim, 2, dtype, device)
        self.proj_out = _plain(cfg['patch_size'] ** 2 * cfg['out_channels'], dim, dtype, device)
        for name, p in self.named_parameters():
            p.original_name = name   # models/qwen_image.py:281-282


# =====================================================================================================================
# pipeline layers (models/qwen_image.py:519-605)
# =====================================================================================================================
class InitialLayer(nn.Module):
    def __init__(self, img_in, txt_norm, txt_in, time_text_embed, axes_dim):
        super().__init__()
        self.img_in, self.txt_norm, self.txt_in, self.time_text_embed = img_in, txt_norm, txt_in, time_text_embed
        self.axes_dim = axes_dim

    def forward(self, inputs):
        for item in inputs:
            if torch.is_floating_point(item):
                item.requires_grad_(True)
        hidden_states, encoder_hidden_states, attention_mask, timestep, img_shapes, txt_seq_lens, *extra = inputs
        hidden_states = linear(hidden_states, self.img_in)
        timestep = timestep.to(torch.bfloat16)
        encoder_hidden_states = linear(self.txt_norm(encoder_hidden_states), self.txt_in)
        temb = self.time_text_embed(timestep)
        shapes = img_shapes.tolist()           # host sync, as in the reference (:535-536)
        lens = txt_seq_lens.tolist()
        vid_freqs, txt_freqs = qwen_rope_tables([tuple(s) for s in shapes[0]], max(lens), self.axes_dim,
                                                device=hidden_states.device)
        Lt = encoder_hidden_states.shape[1]
        # The per-sample prompt lengths travel with the tuple as one int32 tensor (LAST element; `img_seq_len` of the Edit
        # variant is int64) — always, so that every micro-batch of a step has the same tuple structure (the one holding
        # the longest prompt is not padded, the others are).  The block layers read it once per micro-batch and stage.
        text_mask = attention_mask.reshape(attention_mask.shape[0], -1)[:, :Lt]
        key_lens = text_mask.sum(dim=1).to(torch.int32)
        key_lens._dpipe_lens = key_lens.tolist()
        if min(key_lens._dpipe_lens) < Lt and not bool((text_mask.int().diff(dim=1) <= 0).all()):
            raise NotImplementedError('key mask with holes inside the prompt (only trailing padding is supported)')
        extra = list(extra) + [key_lens]
        return make_contiguous(hidden_states, encoder_hidden_states, attention_mask, temb, vid_freqs, txt_freqs) + tuple(extra)


class TransformerLayer(nn.Module):
    def __init__(self, block, block_idx):
        super().__init__()
        self.block = block
        self.block_idx = block_idx

    def forward(self, inputs):
        hidden_states, encoder_hidden_states, attention_mask, temb, vid_freqs, txt_freqs, *extra = inputs
        joint = torch.cat([txt_freqs, vid_freqs], dim=1)           # [2, Lt + Li, 128], order [text, image]
        txt_lens = None
        if extra and extra[-1].dtype == torch.int32:               # prompt lengths (InitialLayer)
            # one host read per micro-batch and stage, not per layer: the same tensor object flows through every layer of
            # a stage, so the decoded lengths are parked on it
            kl = extra[-1]
            lens = getattr(kl, '_dpipe_lens', None)
            if lens is None:
                lens = kl._dpipe_lens = kl.tolist()
            if min(lens) < encoder_hidden_states.shape[1]:         # some prompt is padded: attend per sample over valid rows
                txt_lens = lens
        encoder_hidden_states, hidden_states = self.block(
            hidden_states=hidden_states, encoder_hidden_states=encoder_hidden_states, temb=temb,
            image_rotary_emb=(joint[0], joint[1]), txt_lens=txt_lens)
        return make_contiguous(hidden_states, encoder_hidden_states, attention_mask, temb, vid_freqs, txt_freqs) + tuple(extra)


class FinalLayer(nn.Module):
    def __init__(self, norm_out, proj_out):
        super().__init__()
        self.norm_out, self.proj_out = norm_out, proj_out

    def forward(self, inputs):
        hidden_states, encoder_hidden_states, attention_mask, temb, vid_freqs, txt_freqs, *extra = inputs
        # With Qwen-Image-Edit control latents the reference slices the prediction to `extra[0][0].item()` tokens here
        # (:600-603, a host sync); the loss below keeps the first target.shape[1] tokens instead (shape metadata only).
        hidden_states = AdaLNContinuousFn.apply(hidden_states, temb, self.norm_out.linear)
        return linear(hidden_states, self.proj_out)


# =====================================================================================================================
# the plugin
# =====================================================================================================================
def pack_latents(x):
    """diffusers QwenImagePipeline._pack_latents on [bs, C, 1, h, w] (models/qwen_image.py:415)."""
    b, c = x.shape[0], x.shape[1]
    h, w = x.shape[-2], x.shape[-1]
    return x.reshape(b, c, h // 2, 2, w // 2, 2).permute(0, 2, 4, 1, 3, 5).reshape(b, (h // 2) * (w // 2), c * 4)


class QwenImagePipeline(PluginSurface):
    """Mirror of the reference QwenImagePipeline's training-side surface (models/qwen_image.py:177-517).  VAE, the
    Qwen2.5-VL text encoder and latent caching are outside the hot path (SURVEY.md section 8) and are not provided;
    `prepare_inputs` consumes the same cached tensors (`latents`, `prompt_embeds`, `mask`, optional `control_latents`)."""
    name = 'qwen_image'
    checkpointable_layers = ['TransformerLayer']
    adapter_target_modules = ['QwenImageTransformerBlock']
    framerate = None
    pixels_round_to_multiple = 16

    def __init__(self, config, device='cuda'):
        self.config = config
        self.model_config = config['model']
        dtype = self.model_config.get('dtype', torch.bfloat16)
        if isinstance(dtype, str):
            dtype = {'bfloat16': torch.bfloat16, 'float16': torch.float16, 'float32': torch.float32}[dtype]
        if dtype != torch.bfloat16:
            raise NotImplementedError('the sm_90a Qwen-Image path computes in bf16 (model.dtype must be bfloat16)')
        tcfg = self.model_config.get('transformer_config', None)
        if isinstance(tcfg, str):
            with open(tcfg) as f:
                tcfg = json.load(f)
        self.tcfg = dict(QWEN_IMAGE_CONFIG, **(tcfg or {}))
        device = self.model_config.get("device", device)      # (tests: "cpu" with the kernel test doubles)
        self.dtype, self.device = dtype, device
        self.pipeline_model = None
        self.model_engine = None
        self.adapter_config = None
        self.transformer = None
        if not self.model_config.get('lazy_layers', False):
            self.transformer = QwenImageTransformer2DModel(tcfg, dtype=dtype, device=device)
            if path := self.model_config.get('transformer_path', None):
                self.load_transformer_weights(path)
            self.transformer.train()

    def load_transformer_weights(self, path):
        from .flux import FluxPipeline
        FluxPipeline.load_transformer_weights(self, path)

    def load_diffusion_model(self):
        pass

    def save_model(self, save_dir, state_dict):
        """models/qwen_image.py:296-297"""
        from .flux import FluxPipeline
        FluxPipeline.write_model_file(save_dir, state_dict)

    def configure_adapter(self, adapter_config):
        from .flux import FluxPipeline
        FluxPipeline.configure_adapter(self, adapter_config)

    def _adapt(self, module, dev):
        from .flux import FluxPipeline
        return FluxPipeline._adapt(self, module, dev)

    def load_adapter_weights(self, adapter_path):
        """models/base.py:367-388 (`[adapter] init_from_existing`)"""
        from .flux import FluxPipeline
        FluxPipeline.load_adapter_weights(self, adapter_path)

    def save_adapter(self, save_dir, peft_state_dict):
        """models/qwen_image.py:290-294 (ComfyUI format: keys prefixed with diffusion_model.)"""
        from .flux import FluxPipeline
        FluxPipeline.write_peft_config(self, save_dir, peft_state_dict)
        FluxPipeline.write_adapter_file(save_dir, {'diffusion_model.' + k: v for k, v in peft_state_dict.items()})

    def get_param_groups(self, parameters):
        return [{'params': parameters}]

    def model_specific_dataset_config_validation(self, dataset_config):
        pass

    # ---- data -> model inputs (models/qwen_image.py:394-488) ----
    def prepare_inputs(self, inputs, timestep_quantile=None):
        latents = inputs['latents'].float()
        prompt_embeds = inputs['prompt_embeds']
        mask = inputs['mask']
        device = latents.device
        attn_mask_list = [torch.ones(e.size(0), dtype=torch.bool, device=device) for e in prompt_embeds]
        max_seq_len = max(e.size(0) for e in prompt_embeds)
        prompt_embeds = torch.stack([torch.cat([u, u.new_zeros(max_seq_len - u.size(0), u.size(1))]) for u in prompt_embeds])
        prompt_embeds_mask = torch.stack([torch.cat([u, u.new_zeros(max_seq_len - u.size(0))]) for u in attn_mask_list])
        max_text_len = max_seq_len     # == prompt_embeds_mask.sum(1).max() (:409), known without a device read
        bs, channels, num_frames, h, w = latents.shape
        assert channels == self.tcfg['in_channels'] // 4
        latents = pack_latents(latents)
        if mask is not None:
            mask = mask.unsqueeze(1).expand((-1, channels, -1, -1))
            mask = torch.nn.functional.interpolate(mask, size=(h, w), mode='nearest-exact').unsqueeze(2)
            mask = pack_latents(mask)
        method = self.model_config.get('timestep_sample_method', 'logit_normal')
        if method == 'logit_normal':
            dist = torch.distributions.normal.Normal(0, 1)
        elif method == 'uniform':
            dist = torch.distributions.uniform.Uniform(0, 1)
        else:
            raise NotImplementedError()
        if timestep_quantile is not None:
            t = dist.icdf(torch.full((bs,), timestep_quantile, device=device))
        else:
            t = dist.sample((bs,)).to(device)
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
            x_t, target = ops.noise_on_device(x_1, x_0, t, False, self.device)     # latents are already packed here
        else:
            te = t.view(-1, 1, 1)
            x_t = (1 - te) * x_1 + te * x_0
            target = x_0 - x_1
        img_shapes = [(1, h // 2, w // 2)]
        if 'control_latents' in inputs:
            control = pack_latents(inputs['control_latents'].float())
            assert control.shape == latents.shape, (control.shape, latents.shape)
            extra = (torch.tensor(x_t.shape[1], device=device).repeat((bs,)),)
            x_t = torch.cat([x_t, control.to(x_t.device)], dim=1)
            img_shapes.append((1, h // 2, w // 2))
        else:
            extra = tuple()
        img_shapes = torch.tensor([img_shapes], dtype=torch.int32, device=device).repeat((bs, 1, 1))
        txt_seq_lens = torch.tensor([max_text_len], dtype=torch.int32, device=device).repeat((bs,))
        img_attention_mask = torch.ones((bs, x_t.shape[1]), dtype=torch.bool, device=device)
        attention_mask = torch.cat([prompt_embeds_mask, img_attention_mask], dim=1).view(bs, 1, 1, -1)
        return (x_t, prompt_embeds, attention_mask, t, img_shapes, txt_seq_lens) + extra, (target, mask)

    # ---- layers / loss ----
    def to_layers(self):
        from .flux import base_storage_dtype
        base_storage_dtype(self.model_config, self.adapter_config is not None)    # float8 base: LoRA runs only
        if self.transformer is None:
            return self._lazy_layers()
        t = self.transformer
        layers = [InitialLayer(t.img_in, t.txt_norm, t.txt_in, t.time_text_embed, t.axes_dim)]
        layers += [TransformerLayer(block, i) for i, block in enumerate(t.transformer_blocks)]
        layers.append(FinalLayer(t.norm_out, t.proj_out))
        return layers

    def _lazy_layers(self):
        """Stage-local construction (20 B parameters): LayerSpecs whose builders run only on the owning stage."""
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

        def build_first(dev=None):
            d = dev or device
            w = InitialLayer(_plain(dim, cfg['in_channels'], dtype, d), _RMSNormW(cfg['joint_attention_dim'], dtype, d),
                             _plain(dim, cfg['joint_attention_dim'], dtype, d), QwenTimestepProjEmbeddings(dim, dtype, d),
                             tuple(cfg['axes_dims_rope']))
            return self._adapt(name_params(w, {'': ''}), dev)

        def build_block(i, dev=None):
            w = TransformerLayer(QwenImageTransformerBlock(dim, heads, 4, dtype, dev or device), i)
            return self._adapt(name_params(w, {'block.': f'transformer_blocks.{i}.'}), dev)

        def build_last(dev=None):
            d = dev or device
            w = FinalLayer(_AdaNorm(dim, 2, dtype, d), _plain(cfg['patch_size'] ** 2 * cfg['out_channels'], dim, dtype, d))
            return self._adapt(name_params(w, {'': ''}), dev)

        def count(fn, *a):
            return sum(p.numel() for p in fn(*a, dev='meta').parameters())

        def spec(cls, fn, *a, n):
            s = LayerSpec(cls, *a)
            s.build = lambda fn=fn, a=a: fn(*a)
            s.param_count = n
            return s
        n_block = count(build_block, 0)
        layers = [spec(InitialLayer, build_first, n=count(build_first))]
        layers += [spec(TransformerLayer, build_block, i, n=n_block) for i in range(cfg['num_layers'])]
        layers.append(spec(FinalLayer, build_last, n=count(build_last)))
        return layers

    def get_loss_fn(self):
        from .flux import FluxPipeline
        return FluxPipeline.get_loss_fn(self)
