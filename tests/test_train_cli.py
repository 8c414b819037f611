"""CPU: the driver's CLI / TOML surface (train.py:41-143, 396-429).  GPU: a two-step end-to-end run of train.py on a small
Flux model with save + resume."""
import json
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import train as T  # noqa: E402


def test_cli_accepts_the_reference_flags():
    a = T.build_parser().parse_args(['--config', 'x.toml', '--deepspeed', '--local_rank', '3', '--resume_from_checkpoint',
                                     '--reset_dataloader', '--master_port', '29999', '--i_know_what_i_am_doing'])
    assert a.config == 'x.toml' and a.local_rank == 3 and a.resume_from_checkpoint is True and a.master_port == 29999
    a = T.build_parser().parse_args(['--config', 'x.toml', '--resume_from_checkpoint', '20250101_00-00-00'])
    assert a.resume_from_checkpoint == '20250101_00-00-00'


def test_flags_of_the_caching_stage_are_refused_not_ignored(tmp_path):
    cfg = tmp_path / 'c.toml'
    cfg.write_text("output_dir = 'x'\n")
    for flag in (['--cache_only'], ['--regenerate_cache'], ['--dump_dataset', str(tmp_path)], ['--test_sample']):
        with pytest.raises(NotImplementedError, match='caching'):
            T.main(['--config', str(cfg)] + flag)


def test_config_defaults_and_batch_tables():
    cfg = T.load_toml(os.path.join(ROOT, 'examples', 'flux_synthetic.toml'))
    cfg = T.set_config_defaults(cfg)
    assert cfg['pipeline_stages'] == 1 and cfg['model']['dtype'] is torch.bfloat16 and cfg['model']['guidance'] == 1.0
    assert cfg['eval_before_first_step'] is True and cfg['logging_steps'] == 1 and cfg['warmup_steps'] == 2
    ds, mbs = T.make_ds_config(cfg)
    assert ds == {'train_micro_batch_size_per_gpu': 1, 'gradient_accumulation_steps': 4, 'gradient_clipping': 1.0,
                  'steps_per_print': 1}
    # the engine keys this repo adds to the TOML surface (INTEGRATION.md) reach the engine config; absent keys add nothing
    ds2, _ = T.make_ds_config(dict(cfg, pipeline_schedule='zb', stage_link='dist', zb_max_inflight=6, dp_overlap=False))
    assert ds2['pipeline_schedule'] == 'zb' and ds2['stage_link'] == 'dist' and ds2['zb_max_inflight'] == 6 and ds2['dp_overlap'] is False
    assert T.batch_size_table([[512, 4], [1024, 1]], {None: 1}) == {512: 4, 1024: 1}
    assert T.batch_size_table(None, {None: 3}) == {None: 3}
    with pytest.raises(AssertionError):
        T.set_config_defaults({'model': {'dtype': 'bfloat16'}})          # save_every_n_* is mandatory (train.py:95)
    c = T.set_config_defaults({'save_every_n_epochs': 1, 'model': {'dtype': 'bfloat16'}, 'adapter': {'type': 'lora', 'rank': 16}})
    assert c['adapter'] == {'type': 'lora', 'rank': 16, 'alpha': 16, 'dtype': torch.bfloat16, 'dropout': 0.0}   # train.py:115-133
    with pytest.raises(NotImplementedError):      # alpha is forced to rank
        T.set_config_defaults({'save_every_n_epochs': 1, 'model': {'dtype': 'bfloat16'}, 'adapter': {'type': 'lora', 'rank': 8, 'alpha': 4}})
    with pytest.raises(NotImplementedError):
        T.set_config_defaults({'save_every_n_epochs': 1, 'model': {'dtype': 'bfloat16'}, 'adapter': {'type': 'lokr', 'rank': 8}})


@pytest.mark.gpu
def test_train_two_steps_save_and_resume(tmp_path):
    tcfg = {'num_attention_heads': 2, 'num_layers': 1, 'num_single_layers': 1, 'joint_attention_dim': 64,
            'pooled_projection_dim': 32}
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
max_steps = 2
eval_before_first_step = false
[model]
type = 'flux'
dtype = 'bfloat16'
transformer_config = {{ num_attention_heads = 2, num_layers = 1, num_single_layers = 1, joint_attention_dim = 64, pooled_projection_dim = 32 }}
[optimizer]
type = 'adamw'
lr = 1e-4
betas = [0.9, 0.99]
""")
    run_dir = T.main(['--config', str(cfgp)])
    lines = [json.loads(l) for l in open(os.path.join(run_dir, 'metrics.jsonl'))]
    losses = [l['value'] for l in lines if l['tag'] == 'train/loss']
    assert len(losses) == 2 and all(v == v and v < 100 for v in losses)
    assert os.path.exists(os.path.join(run_dir, 'latest'))
    # resume: continues at step 3 and stops immediately at max_steps... raise the limit to run one more
    cfgp.write_text(cfgp.read_text().replace('max_steps = 2', 'max_steps = 3'))
    run_dir2 = T.main(['--config', str(cfgp), '--resume_from_checkpoint'])
    assert run_dir2 == run_dir
    lines = [json.loads(l) for l in open(os.path.join(run_dir, 'metrics.jsonl'))]
    assert [l['x'] for l in lines if l['tag'] == 'train/loss'] == [1, 2, 3]


@pytest.mark.parametrize('kind,example', [('flux', 'flux_synthetic.toml'), ('qwen_image', 'qwen_image_synthetic.toml'),
                                          ('wan', 'wan_synthetic.toml')])
def test_model_registry_and_synthetic_examples_feed_prepare_inputs(kind, example):
    """every model family with an sm_90a path is reachable from the TOML surface, and its synthetic cached examples have
    the keys / shapes its prepare_inputs consumes (CPU: lazy layers, no kernels)"""
    from diffusion_pipe_b200 import data_feed
    cfg = T.set_config_defaults(T.load_toml(os.path.join(ROOT, 'examples', example)))
    assert cfg['model']['type'] == kind and kind in T.MODEL_TYPES
    cfg['model']['lazy_layers'] = True
    import importlib
    mod, cls = T.MODEL_TYPES[kind]
    model = getattr(importlib.import_module(mod), cls)(cfg, device='cpu')
    syn = {'model': kind, 'num_examples': 4, 'resolution': 128, 'frames': 9, 'text_len': 16, 't5_dim': 64, 'clip_dim': 32,
           'text_dim': 64}
    exs = T.synthetic_examples(syn)
    assert len(exs) == 4
    batch = data_feed.BatchedDataset.collate(exs[:2])
    feats, (target, mask) = model.prepare_inputs(batch)
    assert mask is None and target.shape[0] == 2
    micro = data_feed.split_batch((feats, (target, mask)), 2)
    assert len(micro) == 2 and all(torch.is_tensor(t) for t in micro[0][0])      # None fields became empty tensors
    specs = model.to_layers()
    assert len(specs) == {'flux': 59, 'qwen_image': 62, 'wan': 42}[kind]
    with pytest.raises(NotImplementedError):
        T.make_model({'model': {'type': 'sdxl'}})


def test_train_cli_end_to_end_on_kernel_doubles(tmp_path, monkeypatch):
    """CPU: the whole driver — TOML -> model -> engine -> train loop -> Saver export -> checkpoint -> resume — on a small
    Flux model with the kernel wrappers replaced by the PyTorch test doubles (the GPU variant below uses the kernels)"""
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import kernel_doubles
    from diffusion_pipe_b200 import ops
    kernel_doubles.install(monkeypatch, ops)
    ds = tmp_path / 'ds.toml'
    ds.write_text("[synthetic]\nnum_examples = 8\nresolution = 128\ntext_len = 32\nt5_dim = 64\nclip_dim = 32\n")

    def write_cfg(max_steps, adapter=''):
        cfgp = tmp_path / 'cfg.toml'
        cfgp.write_text(f"""
output_dir = '{tmp_path}/runs'
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
{adapter}
[optimizer]
type = 'adamw'
lr = 1e-4
betas = [0.9, 0.99]
""")
        return cfgp
    cfgp = write_cfg(2)
    run_dir = T.main(['--config', str(cfgp)])
    lines = [json.loads(l) for l in open(os.path.join(run_dir, 'metrics.jsonl'))]
    losses = [l['value'] for l in lines if l['tag'] == 'train/loss']
    assert len(losses) == 2 and all(v == v and v < 100 for v in losses)
    assert os.path.exists(os.path.join(run_dir, 'latest'))
    # the Saver exported the full model at step 2 (utils/saver.py:87-106): one file, reference parameter names, the TOML
    from safetensors.torch import load_file
    sd = load_file(os.path.join(run_dir, 'step2', 'model.safetensors'))
    # ... in the BFL / ComfyUI layout the reference's Flux export uses (models/flux.py:257-288): fused [q; k; v] per stream
    assert 'double_blocks.0.img_attn.qkv.weight' in sd and 'single_blocks.0.linear2.weight' in sd and 'img_in.weight' in sd
    assert sd['double_blocks.0.img_attn.qkv.weight'].shape == (768, 256)
    assert os.path.exists(os.path.join(run_dir, 'step2', 'cfg.toml')) and not os.path.exists(os.path.join(run_dir, 'step2', 'tmp'))
    # resume continues at step 3
    write_cfg(3)
    run_dir2 = T.main(['--config', str(cfgp), '--resume_from_checkpoint'])
    assert run_dir2 == run_dir
    lines = [json.loads(l) for l in open(os.path.join(run_dir, 'metrics.jsonl'))]
    assert [l['x'] for l in lines if l['tag'] == 'train/loss'] == [1, 2, 3]
    assert os.path.exists(os.path.join(run_dir, 'step3', 'model.safetensors'))
    # a LoRA run exports only the adapter factors
    cfgp = write_cfg(1, "[adapter]\ntype = 'lora'\nrank = 16\n")
    (tmp_path / 'runs2').mkdir()
    cfgp.write_text(cfgp.read_text().replace(f"{tmp_path}/runs'", f"{tmp_path}/runs2'"))
    run_dir3 = T.main(['--config', str(cfgp)])
    ad = load_file(os.path.join(run_dir3, 'step1', 'pytorch_lora_weights.safetensors'))      # diffusers' save_lora_weights layout (models/flux.py:231-236)
    assert ad and all('.lora_A.' in k or '.lora_B.' in k for k in ad)
    assert 'transformer.transformer_blocks.0.attn.to_q.lora_A.weight' in ad and ad['transformer.transformer_blocks.0.attn.to_q.lora_A.weight'].shape == (16, 256)
    # ... and runs on a float8 base when [model] asks for it (reference: transformer_dtype = 'float8'), checkpoint + resume included
    cfgp = write_cfg(2, "[adapter]\ntype = 'lora'\nrank = 16\n")
    (tmp_path / 'runs3').mkdir()
    cfgp.write_text(cfgp.read_text().replace(f"{tmp_path}/runs'", f"{tmp_path}/runs3'").replace("dtype = 'bfloat16'\n", "dtype = 'bfloat16'\ntransformer_dtype = 'float8'\n", 1))
    run_dir4 = T.main(['--config', str(cfgp)])
    lines = [json.loads(l) for l in open(os.path.join(run_dir4, 'metrics.jsonl'))]
    assert [l['x'] for l in lines if l['tag'] == 'train/loss'] == [1, 2]
    assert os.path.exists(os.path.join(run_dir4, 'step2', 'pytorch_lora_weights.safetensors'))
    cfgp.write_text(cfgp.read_text().replace('max_steps = 2', 'max_steps = 3'))
    assert T.main(['--config', str(cfgp), '--resume_from_checkpoint']) == run_dir4
    lines = [json.loads(l) for l in open(os.path.join(run_dir4, 'metrics.jsonl'))]
    assert [l['x'] for l in lines if l['tag'] == 'train/loss'] == [1, 2, 3]
    # ... and a new run can start from a saved adapter ([adapter] init_from_existing, train.py:534-535)
    cfgp = write_cfg(1, f"[adapter]\ntype = 'lora'\nrank = 16\ninit_from_existing = '{run_dir4}/step3'\n")
    (tmp_path / 'runs4').mkdir()
    cfgp.write_text(cfgp.read_text().replace(f"{tmp_path}/runs'", f"{tmp_path}/runs4'"))
    run_dir5 = T.main(['--config', str(cfgp)])
    assert os.path.exists(os.path.join(run_dir5, 'step1', 'pytorch_lora_weights.safetensors'))


def test_optimizer_factory_follows_the_reference_rules():
    """train.py:650-663,789-813: beta2 from `beta2_half_life` uses the GLOBAL batch size; 1-D parameters get no weight decay;
    a stage without trainable parameters gets no optimizer; optimizers that are not torch-native are refused, not aliased"""
    class M:
        def get_param_groups(self, params):
            return [{'params': params}]
    w, b = torch.nn.Parameter(torch.zeros(4, 4)), torch.nn.Parameter(torch.zeros(4))
    cfg = {'optimizer': {'type': 'AdamW', 'lr': 1e-4, 'betas': [0.9, 0.99], 'weight_decay': 0.01, 'beta2_half_life': 64}}
    opt = T.make_optimizer_factory(cfg, M(), global_batch_size=16)([w, b])
    assert opt.param_groups[0]['betas'] == (0.9, 0.5 ** (16 / 64))
    assert [g['weight_decay'] for g in opt.param_groups] == [0.01, 0] and opt.param_groups[1]['params'][0] is b
    assert cfg['optimizer']['betas'] == [0.9, 0.99]                       # the config is not edited in place
    assert T.make_optimizer_factory(cfg, M())([]) is None
    with pytest.raises(NotImplementedError):
        T.make_optimizer_factory({'optimizer': {'type': 'stableadamw', 'lr': 1e-4}}, M())([w])
    sgd = T.make_optimizer_factory({'optimizer': {'type': 'sgd', 'lr': 0.1}}, M())([w])
    assert isinstance(sgd, torch.optim.SGD)


def test_train_cli_trains_from_a_cache_the_reference_wrote(tmp_path, monkeypatch, golden_dir):
    """[[directory]] cache_dir = ...: the examples come from tests/golden/ref_cache/, written by the reference's own
    utils/cache.py — the caching stage is unchanged, the hot path consumes its files"""
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import kernel_doubles
    from diffusion_pipe_b200 import ops
    kernel_doubles.install(monkeypatch, ops)
    ds = tmp_path / 'ds.toml'
    ds.write_text(f"[[directory]]\ncache_dir = '{golden_dir}/ref_cache'\nnum_repeats = 1\n")
    cfgp = tmp_path / 'cfg.toml'
    cfgp.write_text(f"""
output_dir = '{tmp_path}/runs'
dataset = '{ds}'
epochs = 2
micro_batch_size_per_gpu = 1
gradient_accumulation_steps = 2
save_every_n_epochs = 1
eval_before_first_step = false
[model]
type = 'flux'
dtype = 'bfloat16'
device = 'cpu'
transformer_config = {{ num_attention_heads = 2, num_layers = 1, num_single_layers = 1, joint_attention_dim = 32, pooled_projection_dim = 16 }}
[optimizer]
type = 'adamw'
lr = 1e-4
""")
    run_dir = T.main(['--config', str(cfgp)])
    lines = [json.loads(l) for l in open(os.path.join(run_dir, 'metrics.jsonl'))]
    # 5 cached examples, global batch 2 -> 2 steps per epoch (the remainder is dropped, utils/dataset.py:350-360), 2 epochs
    assert [l['x'] for l in lines if l['tag'] == 'train/loss'] == [1, 2, 3, 4]
    assert os.path.exists(os.path.join(run_dir, 'epoch1', 'model.safetensors')) and os.path.exists(os.path.join(run_dir, 'epoch2', 'model.safetensors'))


def test_every_example_config_builds_its_model_plan():
    """examples/*.toml (the non-dataset ones): defaults, model dispatch, adapter configuration and the (lazy) layer plan are
    consistent — no parameters are materialised"""
    import glob
    seen = 0
    for path in sorted(glob.glob(os.path.join(ROOT, 'examples', '*.toml'))):
        raw = T.load_toml(path)
        if 'model' not in raw:
            continue                                   # a dataset file
        cfg = T.set_config_defaults(raw)
        cfg['model']['lazy_layers'] = True
        cfg['model']['device'] = 'cpu'
        model = T.make_model(cfg)
        if 'adapter' in cfg:
            model.configure_adapter(cfg['adapter'])
        specs = model.to_layers()
        assert len(specs) >= 3 and all(hasattr(s, 'build') for s in specs), path
        assert os.path.exists(os.path.join(ROOT, cfg['dataset'])), path
        seen += 1
    assert seen >= 5


def test_unsupported_adapter_options_are_refused_and_harmless_keys_are_tolerated():
    base = {'save_every_n_epochs': 1, 'model': {'dtype': 'bfloat16'}}
    for k, v in (('exclude_modules', ['to_q']), ('fuse_adapters', [{'path': 'x'}])):
        with pytest.raises(NotImplementedError):
            T.set_config_defaults(dict(base, model={'dtype': 'bfloat16'}, adapter={'type': 'lora', 'rank': 8, k: v}))
    cfg = T.set_config_defaults(dict(base, model={'dtype': 'bfloat16'}, blocks_to_swap=20, compile=True, monitoring={'enable_wandb': True},
                                     adapter={'type': 'lora', 'rank': 8, 'exclude_modules': None}))
    assert cfg['adapter']['alpha'] == 8 and cfg['compile'] is True
