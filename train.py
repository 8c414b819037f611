#!/usr/bin/env python
"""train.py — the reference's training driver surface (train.py:41-143, 276-974) over the H100-native engine.

    torchrun --nproc-per-node N train.py --config examples/flux_synthetic.toml        (or `deepspeed --num_gpus=N train.py --deepspeed --config ...`)

Same CLI flags and TOML keys as the reference for everything on the hot path (SURVEY.md Appendix B): the model table,
`pipeline_stages`, `micro_batch_size_per_gpu` (int or [[res, bs], ...]), `gradient_accumulation_steps`,
`gradient_clipping`, `partition_method` / `partition_split`, `[optimizer]` (type adamw / adamw_optimi-style kwargs,
`betas`, `weight_decay`, `eps`, `lr`), `lr_scheduler`, `warmup_steps`, `epochs`, `max_steps`, `save_every_n_*`,
`checkpoint_every_n_minutes`, `--resume_from_checkpoint`, `--reset_dataloader`, `--reset_optimizer`.

What is deliberately NOT here (out of the hot path, SURVEY.md section 8): VAE / text-encoder caching of a raw image
folder.  The `dataset` TOML therefore points at already-cached examples:
    [[directory]]   path = "/data/cache.pt"     # torch.save(list of dicts: latents [16,h,w], t5_embed [512,4096], clip_embed [768], mask|None)
or  [synthetic]     num_examples = 64, resolution = 1024      # random latents / embeddings of the named shape
"""
import argparse
import glob
import json
import os
import random
import time
from datetime import datetime, timezone

import torch

try:
    import toml
except ImportError:  # pragma: no cover
    toml = None
    import tomllib

from diffusion_pipe_b200 import data_feed
from diffusion_pipe_b200.pipe import ManualPipelineModule, dist, initialize

TIMESTEP_QUANTILES_FOR_EVAL = [0.1, 0.2, 0.3, 0.4, 0.5, 0.6, 0.7, 0.8, 0.9]
DTYPE_MAP = {'float32': torch.float32, 'float16': torch.float16, 'bfloat16': torch.bfloat16,
             'float8': torch.float8_e4m3fn, 'float8_e4m3fn': torch.float8_e4m3fn, 'float8_e5m2': torch.float8_e5m2}


def build_parser():
    p = argparse.ArgumentParser()
    p.add_argument('--config', help='Path to TOML configuration file.')
    p.add_argument('--local_rank', type=int, default=-1, help='local rank passed from distributed launcher')
    p.add_argument('--resume_from_checkpoint', nargs='?', const=True, default=None)
    p.add_argument('--reset_dataloader', action='store_true')
    p.add_argument('--reset_optimizer', action='store_true')
    p.add_argument('--reset_optimizer_params', action='store_true')
    p.add_argument('--regenerate_cache', action='store_true')
    p.add_argument('--cache_only', action='store_true')
    p.add_argument('--trust_cache', action='store_true')
    p.add_argument('--i_know_what_i_am_doing', action='store_true')
    p.add_argument('--master_port', type=int, default=29500)
    p.add_argument('--dump_dataset', default=None)
    p.add_argument('--test_sample', action='store_true')
    # accepted and ignored: the reference adds these through deepspeed.add_config_arguments (train.py:57)
    p.add_argument('--deepspeed', action='store_true')
    p.add_argument('--deepspeed_config', default=None)
    return p


def load_toml(path):
    if toml is not None:
        with open(path) as f:
            return json.loads(json.dumps(toml.load(f)))
    with open(path, 'rb') as f:
        return json.loads(json.dumps(tomllib.load(f)))


def set_config_defaults(config):
    """train.py:93-143."""
    assert 'save_every_n_epochs' in config or 'save_every_n_steps' in config or 'save_every_n_examples' in config
    config.setdefault('pipeline_stages', 1)
    config.setdefault('activation_checkpointing', False)
    config.setdefault('reentrant_activation_checkpointing', False)
    if config['activation_checkpointing'] == 'unsloth':
        config['reentrant_activation_checkpointing'] = True
    config.setdefault('warmup_steps', 0)
    if 'save_dtype' in config:
        config['save_dtype'] = DTYPE_MAP[config['save_dtype']]
    mc = config['model']
    mc['dtype'] = DTYPE_MAP[mc['dtype']]
    for k in ('transformer_dtype', 'diffusion_model_dtype'):
        if v := mc.get(k, None):
            mc[k] = DTYPE_MAP[v]
    mc.setdefault('guidance', 1.0)
    if 'adapter' in config:                     # train.py:115-133
        ac = config['adapter']
        if 'alpha' in ac:
            raise NotImplementedError('alpha is forced to rank (as in the reference): remove alpha from the [adapter] table')
        if ac['type'] != 'lora':
            raise NotImplementedError(f"adapter type '{ac['type']}': only 'lora' is built for the sm_90a path")
        for k in ('exclude_modules', 'fuse_adapters'):
            if ac.get(k):
                raise NotImplementedError(f"[adapter] {k} is not supported on the sm_90a path: adapters ride the fused GEMM sites of "
                                          'every Linear of the target blocks (models/base.py:263-303 with the default module set)')
        ac['alpha'] = ac['rank']
        ac['dtype'] = DTYPE_MAP[ac['dtype']] if 'dtype' in ac else mc['dtype']
        ac.setdefault('dropout', 0.0)
    config.setdefault('logging_steps', 1)
    config.setdefault('eval_datasets', [])
    config.setdefault('eval_gradient_accumulation_steps', 1)
    config.setdefault('eval_every_n_steps', None)
    config.setdefault('eval_every_n_epochs', None)
    config.setdefault('eval_every_n_examples', None)
    config.setdefault('eval_before_first_step', True)
    config.setdefault('compile', False)
    config.setdefault('x_axis_examples', False)
    return config


def batch_size_table(v, default):
    """int | [[res, bs], ...] -> {None: bs} | {res: bs}   (train.py:396-418)."""
    if v is None:
        return dict(default)
    if isinstance(v, int):
        return {None: v}
    return {x[0]: x[1] for x in v}


def make_ds_config(config):
    mbs = batch_size_table(config.get('micro_batch_size_per_gpu', 1), {None: 1})
    gradient_release = config['optimizer'].get('gradient_release', False)
    ds_config = {
        'train_micro_batch_size_per_gpu': list(mbs.values())[0],
        'gradient_accumulation_steps': config.get('gradient_accumulation_steps', 1),
        'gradient_clipping': 0. if gradient_release else config.get('gradient_clipping', 1.0),
        'steps_per_print': config.get('steps_per_print', 1),
    }
    # engine keys of this repo (not in the reference's TOML surface; INTEGRATION.md section 1): passed through when present
    for key in ('pipeline_schedule', 'stage_link', 'zb_max_inflight', 'zb_costs', 'zb_stage_weights', 'dp_overlap'):
        if key in config:
            ds_config[key] = config[key]
    return ds_config, mbs


# ---------------------------------------------------------------------------------------------------------------------
# cached-example datasets
# ---------------------------------------------------------------------------------------------------------------------
class CachedExamples:
    """One size bucket of already-encoded examples (what utils/cache.py + utils/dataset.py hand to the hot path)."""

    def __init__(self, examples, size_bucket, num_repeats=1):
        self.examples, self.size_bucket, self.num_repeats = examples, tuple(size_bucket), num_repeats

    def __len__(self):
        return int(len(self.examples) * self.num_repeats)

    def __getitem__(self, idx):
        ex = dict(self.examples[idx % len(self.examples)])
        ex.setdefault('mask', None)
        ex.setdefault('caption', '')
        return ex


MODEL_TYPES = {   # config['model']['type'] -> (module, class): the model families with an sm_90a path (train.py:431-535)
    'flux': ('diffusion_pipe_b200.flux', 'FluxPipeline'),
    'qwen_image': ('diffusion_pipe_b200.qwen_image', 'QwenImagePipeline'),
    'wan': ('diffusion_pipe_b200.wan', 'WanPipeline'),
}


def make_model(config):
    import importlib
    model_type = config['model']['type']
    if model_type not in MODEL_TYPES:
        raise NotImplementedError(f"model type '{model_type}': the sm_90a path covers {sorted(MODEL_TYPES)} "
                                  '(SURVEY.md section 8); the other model definitions of the reference are out of scope')
    mod, cls = MODEL_TYPES[model_type]
    return getattr(importlib.import_module(mod), cls)(config)


def synthetic_examples(syn):
    """random cached examples with the keys and shapes the reference's caching step produces for each model family
    (models/flux.py:312-321, models/qwen_image.py:302-318,385-392, models/wan/wan.py:262-330)"""
    n, res = syn.get('num_examples', 16), syn.get('resolution', 1024)
    kind = syn.get('model', 'flux')
    g = torch.Generator().manual_seed(syn.get('seed', 0))
    h = w = res // 8
    if kind == 'flux':
        return [{'latents': torch.randn(16, h, w, generator=g),
                 't5_embed': torch.randn(syn.get('text_len', 512), syn.get('t5_dim', 4096), generator=g).bfloat16(),
                 'clip_embed': torch.randn(syn.get('clip_dim', 768), generator=g).bfloat16(), 'mask': None} for _ in range(n)]
    if kind == 'qwen_image':
        return [{'latents': torch.randn(16, 1, h, w, generator=g),
                 'prompt_embeds': torch.randn(syn.get('text_len', 256), syn.get('text_dim', 3584), generator=g).bfloat16(),
                 'mask': None} for _ in range(n)]
    if kind == 'wan':
        frames = (syn.get('frames', 33) - 1) // 4 + 1            # VAE temporal stride 4 (models/wan/configs.py:63)
        tl = syn.get('text_len', 512)
        exs = [{'latents': torch.randn(16, frames, h, w, generator=g),
                'text_embeddings': torch.randn(tl, syn.get('text_dim', 4096), generator=g).bfloat16(),
                'seq_lens': torch.tensor(syn.get('prompt_len', tl)), 'mask': None} for _ in range(n)]
        if syn.get('i2v', False):        # Wan2.2 I2V (model_type 'i2v_v2'): first-frame conditioning latents
            for ex in exs:
                ex['y'] = torch.randn(16, frames, h, w, generator=g)
        return exs
    raise ValueError(f"[synthetic] model = '{kind}': expected one of flux, qwen_image, wan")


def load_size_buckets(dataset_config):
    out = []
    if syn := dataset_config.get('synthetic', None):
        res = syn.get('resolution', 1024)
        frames = syn.get('frames', 33) if syn.get('model', 'flux') == 'wan' else 1
        out.append(CachedExamples(synthetic_examples(syn), (1.0, res, res, frames), syn.get('num_repeats', 1)))
    for d in dataset_config.get('directory', []):
        if 'cache_dir' in d:
            # the reference's own cache (utils/cache.py), one size-bucket directory `cache_<w>x<h>x<frames>` or a directory
            # of them (`<dataset>/cache/<model name>/`)
            root = d['cache_dir']
            subs = [root] if os.path.isdir(os.path.join(root, 'latents')) else sorted(
                os.path.join(root, n) for n in os.listdir(root) if os.path.isdir(os.path.join(root, n, 'latents')))
            if not subs:
                raise RuntimeError(f'{root}: no size-bucket cache (a directory with latents/ and text_embeddings_*/) found')
            out += [data_feed.ReferenceCacheBucket(sd, d.get('num_repeats', 1)) for sd in subs]
            continue
        exs = torch.load(d['path'], map_location='cpu', weights_only=False)
        by_shape = {}
        for ex in exs:
            c, h, w = ex['latents'].shape[-3:]
            by_shape.setdefault((round(w / h, 3), w * 8, h * 8, 1), []).append(ex)
        for sb, lst in by_shape.items():
            out.append(CachedExamples(lst, sb, d.get('num_repeats', 1)))
    if not out:
        raise RuntimeError('dataset config has neither [synthetic] nor [[directory]] entries')
    return out


def get_most_recent_run_dir(output_dir):
    return list(sorted(glob.glob(os.path.join(output_dir, '*'))))[-1]


def make_optimizer_factory(config, model, global_batch_size=1):
    """train.py:650-815 for the torch-native optimizers; weight-decay / no-weight-decay split as in :789-813;
    `beta2_half_life` (in examples) -> beta2 = 0.5 ** (global_batch_size / half_life) as at :658-663."""
    def factory(params):
        if len(params) == 0:
            return None
        oc = dict(config['optimizer'])
        typ = oc.pop('type').lower()
        oc.pop('gradient_release', None)
        if half_life := oc.pop('beta2_half_life', None):
            b = oc['betas']
            assert len(b) == 2
            oc['betas'] = [b[0], 0.5 ** (global_batch_size / half_life)]
        if 'betas' in oc:
            oc['betas'] = tuple(oc['betas'])
        groups = []
        for pg in model.get_param_groups(params):
            ps = pg.pop('params')
            wd = [p for p in ps if p.ndim != 1]
            nowd = [p for p in ps if p.ndim == 1]
            if wd:
                groups.append(dict(pg, params=wd))
            if nowd:
                groups.append(dict(pg, params=nowd, weight_decay=0))
        if typ in ('adamw', 'adamw_optimi'):            # optimi.AdamW = decoupled AdamW; its Kahan-summation option is not offered
            oc.pop('kahan_sum', None)
            return torch.optim.AdamW(groups, fused=torch.cuda.is_available(), **oc)
        if typ == 'sgd':
            return torch.optim.SGD(groups, **oc)
        raise NotImplementedError(f'optimizer type {typ} is not wired into this driver (third-party optimizers are out of '
                                  'the hot path: pass any torch.optim.Optimizer factory to engine._configure_optimizer)')
    return factory


def evaluate(model_engine, eval_dataloaders, step, egas, log):
    if not eval_dataloaders:
        return
    from diffusion_pipe_b200.data_feed import get_data_iterator_for_step
    cpu_state, cuda_state = torch.get_rng_state(), torch.cuda.get_rng_state() if torch.cuda.is_available() else None
    py_state = random.getstate()
    import numpy as np
    np_state = np.random.get_state()
    seed = dist.get_rank()                                                # train.py:233-238 under isolate_rng()
    random.seed(seed)
    torch.manual_seed(seed)
    np.random.seed(seed)
    start = time.time()
    with torch.no_grad():
        for name, dl in eval_dataloaders.items():
            losses = []
            for q in TIMESTEP_QUANTILES_FOR_EVAL:
                dl.set_eval_quantile(q)
                total, count = 0.0, 0
                while True:
                    model_engine.reset_activation_shape()
                    it = get_data_iterator_for_step(dl, model_engine, num_micro_batches=egas)
                    total += model_engine.eval_batch(it, num_micro_batches=egas).item()
                    dl.sync_epoch()
                    count += 1
                    if dl.epoch == 2:
                        break
                dl.reset()
                losses.append(total / count)
                log(f'{name}/loss_quantile_{q:.2f}', losses[-1], step)
            log(f'{name}/loss', sum(losses) / len(losses), step)
    log('eval/eval_time_sec', time.time() - start, step)
    torch.set_rng_state(cpu_state)
    if cuda_state is not None:
        torch.cuda.set_rng_state(cuda_state)
    random.setstate(py_state)
    np.random.set_state(np_state)


class DeferredScalars:
    """Scalars that live on the device (loss, gradient norm) on their way to the training log without a host sync in the step
    that produced them: push() starts an asynchronous copy into pinned memory, flush() writes out what has arrived."""

    def __init__(self, log):
        self.log = log
        self.pending = []

    def push(self, tag, value, x):
        import torch
        if torch.is_tensor(value) and value.is_cuda:
            host = torch.empty((), dtype=torch.float32, pin_memory=True)
            host.copy_(value.detach().float().reshape(()), non_blocking=True)
            ev = torch.cuda.Event()
            ev.record()
            self.pending.append((tag, host, x, ev))
        else:
            self.pending.append((tag, float(value), x, None))

    def flush(self, keep=0):
        """write everything but the newest `keep` entries (waits for their copies: they were enqueued a step ago)"""
        n = len(self.pending) - keep
        for tag, host, x, ev in self.pending[:max(0, n)]:
            if ev is not None:
                ev.synchronize()
            self.log(tag, float(host), x)
        self.pending = self.pending[max(0, n):]


def main(argv=None):
    args = build_parser().parse_args(argv)
    for flag in ('cache_only', 'regenerate_cache', 'dump_dataset', 'test_sample'):
        if getattr(args, flag):
            # train.py:537-560,897-905: these drive the caching / sampling stages (VAE, text encoders), which stay the reference's
            raise NotImplementedError(f'--{flag} belongs to the latent / text-embedding caching and sampling stages, which stay with the '
                                      "reference's tooling (utils/cache.py is consumed unchanged: [[directory]] cache_dir = ...)")
    config = set_config_defaults(load_toml(args.config))
    world_size = int(os.getenv('WORLD_SIZE', '1'))
    local_rank = args.local_rank if args.local_rank >= 0 else int(os.getenv('LOCAL_RANK', '0'))
    os.environ.setdefault('MASTER_ADDR', '127.0.0.1')
    os.environ.setdefault('MASTER_PORT', str(args.master_port))
    if torch.cuda.is_available():
        torch.cuda.set_device(local_rank)
    if world_size > 1:
        dist.init_distributed()
    is_main = dist.get_rank() == 0

    model = make_model(config)
    is_adapter = False
    if adapter_config := config.get('adapter', None):          # train.py:531-535 (before the layers are built)
        if not hasattr(model, 'configure_adapter'):
            raise NotImplementedError(f"[adapter] is not available for model type '{config['model']['type']}' yet")
        model.configure_adapter(adapter_config)
        is_adapter = True
        if init_from_existing := adapter_config.get('init_from_existing', None):     # train.py:534-535
            model.load_adapter_weights(init_from_existing)

    dataset_config = load_toml(config['dataset'])
    ds_config, micro_batch_size_per_gpu = make_ds_config(config)
    image_mbs = batch_size_table(config.get('image_micro_batch_size_per_gpu'), micro_batch_size_per_gpu)
    eval_mbs = batch_size_table(config.get('eval_micro_batch_size_per_gpu'), micro_batch_size_per_gpu)
    eval_image_mbs = batch_size_table(config.get('eval_image_micro_batch_size_per_gpu'), eval_mbs)
    train_data = data_feed.BatchedDataset(load_size_buckets(dataset_config), dataset_config)
    eval_data_map = {}
    for i, ed in enumerate(config['eval_datasets']):
        name = ed['name'] if isinstance(ed, dict) else f'eval{i}'
        path = ed['config'] if isinstance(ed, dict) else ed
        ecfg = load_toml(path)
        eval_data_map[name] = data_feed.BatchedDataset(load_size_buckets(ecfg), ecfg)

    # run directory (train.py:537-559)
    resume = args.resume_from_checkpoint if args.resume_from_checkpoint is not None else config.get('resume_from_checkpoint', False)
    if resume is True:
        run_dir = get_most_recent_run_dir(config['output_dir'])
    elif isinstance(resume, str):
        run_dir = os.path.join(config['output_dir'], resume)
    else:
        run_dir = os.path.join(config['output_dir'], datetime.now(timezone.utc).strftime('%Y%m%d_%H-%M-%S'))
        if is_main:
            os.makedirs(run_dir, exist_ok=True)
            with open(os.path.join(run_dir, os.path.basename(args.config)), 'w') as f, open(args.config) as src:
                f.write(src.read())
    if world_size > 1:
        holder = [run_dir]
        dist.broadcast_object_list(holder, src=0)
        run_dir = holder[0]

    if config.get('blocks_to_swap', 0) and is_main:                        # train.py:576-583
        print('blocks_to_swap is ignored: block swapping exists to fit 24 GB parts; this engine keeps the whole stage resident '
              '(80 GB HBM per GPU)')
    if 'monitoring' in config and is_main:
        print('[monitoring] (wandb) is ignored: metrics go to <run_dir>/metrics.jsonl')
    layers = model.to_layers()
    extra = {}
    if config['activation_checkpointing']:
        from functools import partial
        extra = {'activation_checkpoint_interval': 1, 'checkpointable_layers': model.checkpointable_layers,
                 'activation_checkpoint_func': partial(torch.utils.checkpoint.checkpoint,
                                                       use_reentrant=config['reentrant_activation_checkpointing'])}
    num_stages = config.get('pipeline_stages', 1)
    pipeline_model = ManualPipelineModule(
        layers=layers, num_stages=num_stages, partition_method=config.get('partition_method', 'parameters'),
        manual_partition_split=config.get('partition_split', None), loss_fn=model.get_loss_fn(), dynamic_shape=True, **extra)
    model.pipeline_model = pipeline_model
    if config['compile']:                                               # train.py:620-621 (a no-op on this engine)
        pipeline_model.compile(dynamic=True)
    parameters_to_train = [p for p in pipeline_model.parameters() if p.requires_grad]
    model_engine, optimizer, _, _ = initialize(args=args, model=pipeline_model, config=ds_config)
    global_batch_size = (model_engine.train_micro_batch_size_per_gpu() * model_engine.gradient_accumulation_steps()
                         * model_engine.grid.get_data_parallel_world_size())
    if is_main:
        print(f'Global batch size = {global_batch_size}')
    if n := config.pop('save_every_n_examples', None):
        config['save_every_n_steps'] = n // global_batch_size
    if n := config.pop('eval_every_n_examples', None):
        config['eval_every_n_steps'] = n // global_batch_size

    model_engine._configure_optimizer(make_optimizer_factory(config, model, global_batch_size), parameters_to_train)
    optimizer = model_engine.optimizer
    model.model_engine = model_engine
    grid = model_engine.grid
    train_data.post_init(grid.get_data_parallel_rank(), grid.get_data_parallel_world_size(), micro_batch_size_per_gpu,
                         model_engine.gradient_accumulation_steps(), image_mbs)
    for ed in eval_data_map.values():
        ed.post_init(grid.get_data_parallel_rank(), grid.get_data_parallel_world_size(), eval_mbs,
                     config['eval_gradient_accumulation_steps'], eval_image_mbs)
    model_engine.communication_data_type = config['model']['dtype']
    train_dataloader = data_feed.PipelineDataLoader(train_data, model_engine, model_engine.gradient_accumulation_steps(), model,
                                                    num_dataloader_workers=config.get('num_dataloader_workers', 0))
    steps_per_epoch = len(train_dataloader) // model_engine.gradient_accumulation_steps()

    if optimizer is not None:
        st = config.get('lr_scheduler', 'constant')
        total = config.get('epochs', 1) * steps_per_epoch
        if st == 'constant':
            sched = torch.optim.lr_scheduler.ConstantLR(optimizer, factor=1.0)
        elif st == 'linear':
            sched = torch.optim.lr_scheduler.LinearLR(optimizer, start_factor=1.0, end_factor=0.0, total_iters=total)
        elif st == 'cosine':
            sched = torch.optim.lr_scheduler.CosineAnnealingLR(optimizer, T_max=total, eta_min=1e-6)
        else:
            raise NotImplementedError(f'Unknown lr_scheduler: {st}')
        if config['warmup_steps'] > 0:
            w = config['warmup_steps']
            warm = torch.optim.lr_scheduler.LinearLR(optimizer, start_factor=1 / w, total_iters=w)
            sched = torch.optim.lr_scheduler.SequentialLR(optimizer, schedulers=[warm, sched], milestones=[w])
        model_engine.lr_scheduler = sched

    step, examples = 1, global_batch_size
    if resume:
        param_groups = optimizer.param_groups.copy() if optimizer is not None else None
        load_path, client_state = model_engine.load_checkpoint(
            run_dir, load_module_strict=False,
            load_lr_scheduler_states='force_constant_lr' not in config and not args.reset_optimizer and not args.reset_optimizer_params,
            load_optimizer_states=not args.reset_optimizer)
        assert load_path is not None
        if args.reset_optimizer_params and optimizer is not None:        # train.py:874-875: keep the TOML's lr / betas / ...
            optimizer.param_groups = param_groups
        if args.reset_dataloader:
            train_dataloader.set_epoch(client_state['custom_loader']['epoch'])
        else:
            train_dataloader.load_state_dict(client_state['custom_loader'])
        step = client_state['step'] + 1
        examples = client_state.get('examples', step * global_batch_size - global_batch_size) + global_batch_size
        if is_main:
            print(f'Resuming training from checkpoint. Resuming at epoch: {train_dataloader.epoch}, step: {step}')
    if 'force_constant_lr' in config and optimizer is not None:
        model_engine.lr_scheduler = torch.optim.lr_scheduler.ConstantLR(optimizer, factor=1.0)
        for pg in optimizer.param_groups:
            pg['lr'] = config['force_constant_lr']

    eval_dataloaders = {name: data_feed.PipelineDataLoader(ed, model_engine, config['eval_gradient_accumulation_steps'], model,
                                                           num_dataloader_workers=0) for name, ed in eval_data_map.items()}
    metrics = []

    def log(tag, value, x):
        if is_main:
            metrics.append({'tag': tag, 'value': float(value), 'x': x})
            with open(os.path.join(run_dir, 'metrics.jsonl'), 'a') as f:
                f.write(json.dumps(metrics[-1]) + '\n')

    from diffusion_pipe_b200.saver import Saver
    saver = Saver(args, config, is_adapter, run_dir, model, train_dataloader, model_engine, pipeline_model)

    if config['eval_before_first_step'] and not resume:
        evaluate(model_engine, eval_dataloaders, 0, config['eval_gradient_accumulation_steps'], log)

    epoch = train_dataloader.epoch
    epoch_loss, num_steps = None, 0
    checkpointed = saved = False
    final_model_name = None
    # SURVEY.md 8(f)4: the reference reads the loss back with `.item()` after every step (train.py:918), a host<->device sync that
    # keeps the next step's first kernels from being enqueued until the last optimizer kernel has finished.  Here the scalars
    # of step s travel to pinned host memory asynchronously and are written to the log once step s+1 has been enqueued — the
    # same numbers against the same x axis, one step later; everything pending is flushed before an evaluation, at the end of
    # an epoch and on exit.  The epoch mean accumulates on the device.
    scalars = DeferredScalars(log)
    while True:                                                          # train.py:915-965
        model_engine.reset_activation_shape()
        iterator = data_feed.get_data_iterator_for_step(train_dataloader, model_engine)
        loss = model_engine.train_batch(iterator)
        epoch_loss = loss.detach().float().clone() if epoch_loss is None else epoch_loss + loss.detach().float()
        num_steps += 1
        train_dataloader.sync_epoch()
        new_epoch, checkpointed, saved = saver.process_epoch(epoch, step, examples)
        finished_epoch = new_epoch != epoch
        x_axis = examples if config['x_axis_examples'] else step
        scalars.flush(keep=0)                                            # step s-1: its copies finished long ago
        if step % config['logging_steps'] == 0:
            scalars.push('train/loss', loss, x_axis)
            if model_engine._grad_norm is not None:
                scalars.push('train/grad_norm', model_engine._grad_norm, x_axis)
        if (config['eval_every_n_steps'] and step % config['eval_every_n_steps'] == 0) or \
                (finished_epoch and config['eval_every_n_epochs'] and epoch % config['eval_every_n_epochs'] == 0):
            scalars.flush(keep=0)
            evaluate(model_engine, eval_dataloaders, x_axis, config['eval_gradient_accumulation_steps'], log)
        if finished_epoch:
            scalars.flush(keep=0)
            log('train/epoch_loss', float(epoch_loss) / num_steps, epoch)
            epoch_loss, num_steps = None, 0
            if new_epoch is None:
                final_model_name = f'epoch{epoch}'
                break
            epoch = new_epoch
        checkpointed, saved = saver.process_step(step, examples)
        if 'max_steps' in config and step >= config['max_steps']:
            final_model_name = f'step{step}'
            break
        step += 1
        examples += global_batch_size
    scalars.flush(keep=0)
    # final training state and model, unless they were just written
    if not checkpointed:
        saver.save_checkpoint(step, examples)
    if not saved:
        saver.save_model(final_model_name)
    if is_main:
        print('TRAINING COMPLETE!')
    return run_dir


if __name__ == '__main__':
    main()
