"""CPU / gloo: the REFERENCE's own driver-side code, unmodified, on top of the new engine — the drop-in boundary B-py.2
(SURVEY.md 8b) exercised by the code that will actually call it:

    utils/saver.py                      imported as it is (module); `deepspeed.comm` -> diffusion_pipe_b200.pipe.dist
    utils/dataset.py:1273-1450          split_batch, PipelineDataLoader, SkipFirstNSampler   (source text)
    train.py:167-173                    get_data_iterator_for_step                            (source text)
    train.py:39,176-242                 evaluate / _evaluate / evaluate_single + utils/isolate_rng.py (source text / module)

They drive diffusion_pipe_b200's engine, PipelineModule and FluxPipeline (kernel wrappers = the CPU test doubles) for a few
optimizer steps with model export, checkpoint and resume, for 1 and 2 pipeline stages, and must give the same losses
and files as this repo's own data_feed.PipelineDataLoader / saver.Saver.

What that code produced (the 'reference' arm) is stored in tests/golden/dropin_golden.pt by tests/golden/make_golden_dropin.py,
which needs /root/reference; the test runs this repo's arm and compares with it.  Two stand-ins only: the reference moves the target
`.to('cuda')` before its p2p send (utils/dataset.py:1399) — redirected to the CPU for the gloo run — and
`deepspeed.utils.logging.logger` is a stdlib logger.
"""
import ast
import importlib.util
import json
import logging
import os
import socket
import sys
import tempfile
import types

import pytest
import torch
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = '/root/reference'      # read by the fixture generator only (load_reference_driver_code)
GOLDEN = os.path.join(HERE, 'golden', 'dropin_golden.pt')
for p in (ROOT, HERE, os.path.join(HERE, 'golden')):
    if p not in sys.path:
        sys.path.insert(0, p)

GAS, STEPS = 2, 3
CFG = {'num_attention_heads': 2, 'num_layers': 1, 'num_single_layers': 1, 'joint_attention_dim': 64, 'pooled_projection_dim': 32}


def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    return port


class _Patch:
    def setattr(self, obj, name, value):
        setattr(obj, name, value)


def load_reference_driver_code():
    from diffusion_pipe_b200.pipe import dist
    ds = types.ModuleType('deepspeed'); ds.__path__ = []
    ds_utils = types.ModuleType('deepspeed.utils'); ds_utils.__path__ = []
    ds_log = types.ModuleType('deepspeed.utils.logging'); ds_log.logger = logging.getLogger('reference')
    utils = types.ModuleType('utils'); utils.__path__ = []
    common = types.ModuleType('utils.common'); common.is_main_process = lambda: dist.get_rank() == 0
    ds.comm = dist
    for n, m in (('deepspeed', ds), ('deepspeed.comm', dist), ('deepspeed.utils', ds_utils), ('deepspeed.utils.logging', ds_log),
                 ('utils', utils), ('utils.common', common)):
        sys.modules[n] = m
    spec = importlib.util.spec_from_file_location('reference_saver', os.path.join(REF, 'utils', 'saver.py'))
    saver = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(saver)
    ns = {'torch': torch, 'dist': dist, 'is_main_process': common.is_main_process}
    tree = ast.parse(open(os.path.join(REF, 'utils', 'dataset.py')).read())
    body = [n for n in tree.body if (isinstance(n, ast.FunctionDef) and n.name == 'split_batch')
            or (isinstance(n, ast.ClassDef) and n.name in ('PipelineDataLoader', 'SkipFirstNSampler'))]
    assert len(body) == 3
    exec(compile(ast.Module(body=body, type_ignores=[]), 'utils/dataset.py', 'exec'), ns)
    tree = ast.parse(open(os.path.join(REF, 'train.py')).read())
    body = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == 'get_data_iterator_for_step']
    exec(compile(ast.Module(body=body, type_ignores=[]), 'train.py', 'exec'), ns)
    # train.py:39,176-242: the evaluation functions (quantile sweep, RNG isolation, block-swap hooks of the plugin)
    import random
    import time
    import numpy as np
    spec = importlib.util.spec_from_file_location('reference_isolate_rng', os.path.join(REF, 'utils', 'isolate_rng.py'))
    iso = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(iso)

    class tqdm:
        def __init__(self, total=None):
            self.total, self.n = total, 0

        def update(self, k):
            self.n += k

        def close(self):
            assert self.n == self.total, (self.n, self.total)      # the reference's own progress arithmetic adds up
    ns.update({'random': random, 'time': time, 'np': np, 'tqdm': tqdm, 'wandb_enable': False, 'wandb': None,
               'empty_cuda_cache': lambda: None, 'isolate_rng': iso.isolate_rng, 'get_rank': dist.get_rank})
    body = [n for n in tree.body if (isinstance(n, ast.FunctionDef) and n.name in ('evaluate_single', '_evaluate', 'evaluate'))
            or (isinstance(n, ast.Assign) and getattr(n.targets[0], 'id', '') == 'TIMESTEP_QUANTILES_FOR_EVAL')]
    assert len(body) == 4
    exec(compile(ast.Module(body=body, type_ignores=[]), 'train.py', 'exec'), ns)
    return saver.Saver, ns['PipelineDataLoader'], ns['get_data_iterator_for_step'], ns['evaluate']


class Batches:
    """the interface both loaders use of the batched dataset: len, item -> one collated global batch, dataset_config"""
    dataset_config = {}

    def __init__(self, n, batch_size):
        g = torch.Generator().manual_seed(7)
        self.items = [{'latents': torch.randn(batch_size, 16, 8, 8, generator=g), 't5_embed': torch.randn(batch_size, 12, 64, generator=g).bfloat16(),
                       'clip_embed': torch.randn(batch_size, 32, generator=g).bfloat16(), 'mask': None} for _ in range(n)]

    def __len__(self):
        return len(self.items)

    def __getitem__(self, i):
        return self.items[i]


def _worker(rank, world, port, which, outdir, resume):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    import kernel_doubles
    from diffusion_pipe_b200 import data_feed, ops
    from diffusion_pipe_b200 import saver as my_saver
    from diffusion_pipe_b200.flux import FluxPipeline
    from diffusion_pipe_b200.pipe import ManualPipelineModule, dist, initialize
    kernel_doubles.install(_Patch(), ops)
    torch.set_num_threads(1)
    dist.init_distributed('gloo')
    real_to = torch.Tensor.to

    def to(self, *a, **k):          # utils/dataset.py:1399 `target.to('cuda')`: there is no CUDA device in this run
        return real_to(self, *tuple('cpu' if x == 'cuda' else x for x in a), **k)
    torch.Tensor.to = to

    torch.manual_seed(0)
    cfgfile = os.path.join(outdir, 'config.toml')
    if rank == 0 and not os.path.exists(cfgfile):
        open(cfgfile, 'w').write('# run config\n')
    config = {'model': {'dtype': 'bfloat16', 'guidance': 1.0, 'device': 'cpu', 'transformer_config': CFG}, 'epochs': 100,
              'save_every_n_steps': 2, 'checkpoint_every_n_epochs': 1}
    model = FluxPipeline(config)
    pm = ManualPipelineModule(layers=model.to_layers(), num_stages=world, partition_method='uniform', loss_fn=model.get_loss_fn(),
                              dynamic_shape=True, device=torch.device('cpu'))
    engine, _, _, _ = initialize(model=pm, config={'train_micro_batch_size_per_gpu': 1, 'gradient_accumulation_steps': GAS,
                                                   'gradient_clipping': 1.0, 'steps_per_print': 0, 'stage_link': 'dist'})
    engine._configure_optimizer(lambda ps: torch.optim.SGD(ps, lr=0.01) if ps else None, [p for p in pm.parameters() if p.requires_grad])
    if engine.is_pipe_parallel:                                   # train.py:821-823
        grid = engine.grid
        engine.first_last_stage_group = dist.new_group(ranks=[grid.pp_group[0], grid.pp_group[-1]])
    if which == 'reference':
        RefSaver, RefLoader, get_iter, ref_evaluate = load_reference_driver_code()
        loader = RefLoader(Batches(2, GAS), engine, GAS, model, num_dataloader_workers=0)
        eval_loader = RefLoader(Batches(2, 1), engine, 1, model, num_dataloader_workers=0)
    else:
        RefSaver, get_iter = my_saver.Saver, data_feed.get_data_iterator_for_step
        loader = data_feed.PipelineDataLoader(Batches(2, GAS), engine, GAS, model, num_dataloader_workers=0)
        eval_loader = data_feed.PipelineDataLoader(Batches(2, 1), engine, 1, model, num_dataloader_workers=0)
    run_dir = os.path.join(outdir, 'run_' + which)
    if rank == 0:
        os.makedirs(run_dir, exist_ok=True)
    dist.barrier()
    args = types.SimpleNamespace(config=cfgfile)
    step, first = 1, 1
    if resume:
        _, client_state = engine.load_checkpoint(run_dir, load_module_strict=False, load_lr_scheduler_states=True, load_optimizer_states=True)
        loader.load_state_dict(client_state['custom_loader'])
        step = first = client_state['step'] + 1
    saver = RefSaver(args, config, False, run_dir, model, loader, engine, pm)
    epoch = loader.epoch
    losses, epochs = [], []
    while step < first + STEPS:                                               # the loop body of train.py:915-962
        engine.reset_activation_shape()
        torch.manual_seed(1000 + step)                                        # (prepare_inputs draws noise: same draws in both runs)
        iterator = get_iter(loader, engine)
        losses.append(engine.train_batch(iterator).item())
        loader.sync_epoch()
        new_epoch, checkpointed, saved = saver.process_epoch(epoch, step, step * GAS)
        epochs.append(loader.epoch)
        if new_epoch != epoch:
            epoch = new_epoch
        saver.process_step(step, step * GAS)
        step += 1
    # evaluation: 9 timestep quantiles x the whole eval set, seeded by rank, RNG state restored afterwards
    scalars = []
    rng_before = torch.get_rng_state().clone()
    if which == 'reference':
        tb = types.SimpleNamespace(add_scalar=lambda tag, value, x: scalars.append((tag, float(value), x)))
        ref_evaluate(model, engine, {'eval0': eval_loader}, tb, step, 1, False)
    else:
        sys.path.insert(0, ROOT)
        import train as my_train
        my_train.evaluate(engine, {'eval0': eval_loader}, step, 1, lambda tag, value, x: scalars.append((tag, float(value), x)))
    assert torch.equal(torch.get_rng_state(), rng_before)
    scalars = [s for s in scalars if s[0] != 'eval/eval_time_sec']
    torch.save({'losses': losses, 'epochs': epochs, 'state': loader.state_dict(), 'eval': scalars},
               os.path.join(outdir, f'{which}_resume{int(resume)}_rank{rank}.pt'))
    dist.barrier()


def _run(world, which, outdir, resume=False):
    mp.spawn(_worker, args=(world, _free_port(), which, outdir, resume), nprocs=world, join=True)
    return [torch.load(os.path.join(outdir, f'{which}_resume{int(resume)}_rank{r}.pt'), weights_only=False) for r in range(world)]


def tensor_summary(t):
    """shape, dtype, float64 sum and sum of squares and the first 8 elements of one exported tensor"""
    f = t.double().reshape(-1)
    return {'shape': list(t.shape), 'dtype': str(t.dtype), 'sum': f.sum().item(), 'sumsq': (f * f).sum().item(),
            'head': f[:8].tolist()}


def run_record(world, which, d):
    """everything the test compares, for one arm at one pipeline depth (the resume leg on the 2-stage pipeline only)"""
    from safetensors.torch import load_file
    rec = {'ranks': _run(world, which, d)}
    run = os.path.join(d, 'run_' + which)
    rec['checkpointed'] = os.path.exists(os.path.join(run, 'latest')) or any(n.startswith('global_step') for n in os.listdir(run))
    rec['step2_config'] = os.path.exists(os.path.join(run, 'step2', 'config.toml'))
    rec['step2_tmp'] = os.path.exists(os.path.join(run, 'step2', 'tmp'))
    rec['export'] = {k: tensor_summary(v) for k, v in sorted(load_file(os.path.join(run, 'step2', 'model.safetensors')).items())}
    if world == 2:
        rec['resume'] = _run(world, which, d, resume=True)
    return json.loads(json.dumps(rec))          # tuples -> lists, as the stored fixture has them


def _close(a, b, rtol=1e-5):
    return abs(a - b) <= rtol * max(abs(a), abs(b), 1e-6)


@pytest.mark.parametrize('world', [1, 2])
def test_reference_loader_and_saver_drive_the_engine(world):
    ref = torch.load(GOLDEN, weights_only=False)[str(world)]
    with tempfile.TemporaryDirectory() as d:
        mine = run_record(world, 'mine', d)
    for r, m in zip(ref['ranks'], mine['ranks'], strict=True):
        assert len(r['losses']) == len(m['losses']) and all(_close(a, b) for a, b in zip(r['losses'], m['losses']))
        assert all(v == v and 0 < v < 100 for v in m['losses'])
        assert r['epochs'] == m['epochs'] == [1, 2, 2]            # 2 batches per epoch: the epoch turns when the last one is RETURNED
        assert r['state'] == m['state']
    # the reference's evaluate() logs on rank 0 only; this repo's log callback is rank-0-gated by its caller
    re_, me = ref['ranks'][0]['eval'], mine['ranks'][0]['eval']
    assert len(re_) == len(me) == 10
    assert all(a[0] == b[0] and a[2] == b[2] and _close(a[1], b[1]) for a, b in zip(re_, me))
    assert [t for t, _, _ in me][:2] == ['eval0/loss_quantile_0.10', 'eval0/loss_quantile_0.20'] and me[-1][0] == 'eval0/loss'
    assert ref['checkpointed'] and mine['checkpointed'] and ref['step2_config'] and mine['step2_config']
    assert not ref['step2_tmp'] and not mine['step2_tmp']
    a, b = ref['export'], mine['export']
    assert set(a) == set(b) and 'double_blocks.0.img_attn.qkv.weight' in a and 'single_blocks.0.linear2.weight' in a   # BFL layout
    for k in a:
        assert a[k]['shape'] == b[k]['shape'] and a[k]['dtype'] == b[k]['dtype'], k
        assert _close(a[k]['sum'], b[k]['sum'], 1e-4) and _close(a[k]['sumsq'], b[k]['sumsq'], 1e-5), k
        assert all(_close(x, y, 1e-5) for x, y in zip(a[k]['head'], b[k]['head'])), k
    if world == 1:
        return                                                      # (the resume leg runs once, on the 2-stage pipeline)
    # resume from the checkpoint the reference's Saver asked the engine to write (end of epoch 1 = step 2)
    for r, m in zip(ref['resume'], mine['resume'], strict=True):
        assert all(_close(x, y) for x, y in zip(r['losses'], m['losses'], strict=True)) and r['state'] == m['state']
    # (The checkpoint sits exactly on the epoch boundary, where the reference's loader has pulled 0 batches of the new
    #  epoch: its `num_batches_pulled - 1` resume rule (utils/dataset.py:1430) then starts from index -1, i.e. replays
    #  the LAST batch first.  data_feed.PipelineDataLoader reproduces that, which is what the equalities above show;
    #  the resumed step therefore differs from the uninterrupted run's step 3 in BOTH implementations.)
    assert mine['resume'][0]['losses'][0] != mine['ranks'][0]['losses'][2]
    assert ref['resume'][0]['losses'][0] != ref['ranks'][0]['losses'][2]
