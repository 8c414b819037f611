"""CPU: the host-side pieces of bench.py the driver's scaling run depends on — the measured-time stage split, the per-layer
weight seeding (same model for every --gpus N) and the reference arm's JSON contract."""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def test_time_balanced_split_prefers_fewer_double_blocks_per_stage():
    import bench
    # Flux-dev: 19 double + 38 single blocks; a double block costs 1.3x a single block in time (the calibration value of the stage split)
    for stages in (2, 4, 8):
        split, stage_ms, blocks = bench.time_balanced_split(19, 38, stages, 1.3 * 30.0, 30.0, 16, (30, 40, 30), 0)
        assert len(split) == stages - 1 and sum(blocks) == 57 and all(b > 0 for b in blocks)
        assert split == sorted(split) and split[0] >= 2 and split[-1] <= 57
        # no stage is more than 12 % above the mean: round 1's count-balanced split put 8 double blocks (+30 %) on stage 0
        assert max(stage_ms) <= 1.12 * sum(stage_ms) / stages, (stages, stage_ms)
    split8, _, blocks8 = bench.time_balanced_split(19, 38, 8, 1.3 * 30.0, 30.0, 16, (30, 40, 30), 0)
    assert blocks8[0] < blocks8[-1]                       # stages made of double blocks hold fewer blocks
    count_split, per_stage = bench.flop_balanced_split(19, 38, 8)
    assert per_stage == [8, 7, 7, 7, 7, 7, 7, 7] and count_split[0] == 9


def test_layer_seeding_gives_the_same_weights_for_any_build_order():
    import bench
    from diffusion_pipe_b200.pipe.module import LayerSpec

    def make_specs():
        return bench.seed_layers([LayerSpec(torch.nn.Linear, 8, 8) for _ in range(4)])
    a = [s.build().weight.detach().clone() for s in make_specs()]
    specs = make_specs()
    torch.manual_seed(999)                                # another rank: other RNG state, builds only the last two layers, in reverse
    b3 = specs[3].build().weight.detach().clone()
    b2 = specs[2].build().weight.detach().clone()
    assert torch.equal(a[3], b3) and torch.equal(a[2], b2) and not torch.equal(a[2], a[3])


def test_reference_arm_is_rank0_only_and_bounded(monkeypatch):
    """--impl reference under torchrun: ranks > 0 exit without work; the line carries the contract keys (the timing itself
    needs minutes of CPU at the real shape: here the sampler is stubbed)"""
    import bench
    monkeypatch.setattr(bench, 'cpu_reference_sample', lambda *a, **k: (1e-3, 'stub sample', 8))
    monkeypatch.setenv('RANK', '1')
    monkeypatch.setattr(sys, 'argv', ['bench.py', '--impl', 'reference', '--gpus', '2'])
    assert bench.main() is None
    monkeypatch.setenv('RANK', '0')
    import io
    import contextlib
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        bench.main()
    line = json.loads(buf.getvalue().strip().splitlines()[-1])
    assert line['impl'] == 'reference' and line['gpu_launches'] == 0 and line['higher_is_better'] is True
    assert line['cpu_baseline']['kind'] == 'port' and line['cpu_baseline']['cores'] == 8 and len(line['cpu_baseline']['min_max']) == 2
    assert line['e2e'] == {'value': line['value'], 'unit': 'samples/s', 'h2d_bytes_per_step': 0, 'd2h_bytes_per_step': 0}
    assert line['metric'].startswith('training samples/sec')


def test_split_from_probe_falls_back_when_the_measurement_is_implausible_or_missing():
    import bench
    good = [4.9, 3.71, 1.455, 2.529, 0.957, 1.137, 1.774, 0.761]                  # the 8-GPU run of round 2
    split, blocks, weights, costs, desc = bench.split_from_probe(good, 19, 38, 8, 16, 0)
    assert blocks == [6, 6, 6, 7, 8, 8, 8, 8] and desc['method'].startswith('measured') and len(weights) == 8
    assert abs(sum(costs) - 100) <= 2 and all(abs(c - r) <= 0.35 * r for c, r in zip(costs, bench.CALIBRATED_FBW))
    bad = [9.476, 3.576, 3.121, 4.831, 0.953, 1.109, 1.71, 0.74]                  # the disturbed 2-GPU probe: 2.65x
    split, blocks, weights, costs, desc = bench.split_from_probe(bad, 19, 38, 2, 16, 0)
    assert blocks == [26, 31] and costs == bench.CALIBRATED_FBW and 'calibrated' in desc['method']
    assert desc['double_over_single'] == bench.CALIBRATED_DOUBLE_OVER_SINGLE
    none = [float('inf')] * 8                                                     # every rank's probe failed
    split, blocks, weights, costs, desc = bench.split_from_probe(none, 19, 38, 4, 16, 0)
    assert sum(blocks) == 57 and costs == bench.CALIBRATED_FBW and all(w >= 1 for w in weights)


def test_the_orders_the_scaling_run_will_execute_are_complete_and_deadlock_free():
    """exactly what `bench.py --gpus N` hands to the engine for N = 2, 3, 4, 8 (zero-bubble order, per-stage weights and F:B:W
    costs from the block-time probe or from the calibrated fallback)"""
    import bench
    from diffusion_pipe_b200.pipe.schedule import ZeroBubbleSchedule
    good = [4.9, 3.71, 1.455, 2.529, 0.957, 1.137, 1.774, 0.761]
    for probe in (good, [float('inf')] * 8):
        for stages in (2, 3, 4, 8):
            _split, blocks, weights, costs, _ = bench.split_from_probe(probe, 19, 38, stages, 16, 0)
            assert sum(blocks) == 57 and len(weights) == stages
            for st in range(stages):
                seq = [(c.name, getattr(c, 'micro_batch_id', None))
                       for t in ZeroBubbleSchedule(16, stages, st, costs, None, weights).steps() for c in t]
                for kind in ('ForwardPass', 'BackwardInput', 'BackwardWeight'):
                    assert [mb for n, mb in seq if n == kind] == list(range(16)), (stages, st, kind)
                held = peak = 0
                for n, _ in seq:
                    held += (n == 'ForwardPass') - (n == 'BackwardWeight')
                    peak = max(peak, held)
                assert peak <= 2 * stages, (stages, st, peak)          # IpcLink sizes its mailboxes for 2 x stages slots
            ms = ZeroBubbleSchedule(16, stages, 0, costs, None, weights).simulated_makespan()
            work = 16 * sum(costs) * max(weights)
            assert ms > 0 and work / ms > 0.80, (stages, work / ms)     # the joint replay completes; bubble below 20 %
