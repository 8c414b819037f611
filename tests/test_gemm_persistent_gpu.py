"""GPU: the persistent wgmma GEMM, where one CTA per SM walks several tiles, element by element against the fp64
references of tests/gemm_attn_refs.py.

Grids of more tiles than SMs give each CTA several tiles in a row, so the ring's barrier phases run on across tiles and
each warpgroup's epilogue buffer is reused while the producer already loads the next tile.  The last tile of the grid
(the last of its CTA) carries both an M tail and an N tail.  Small-integer inputs hold the outputs to exact bits where
no transcendental follows; every case is launched twice and must repeat its bits."""
import pytest
import torch

from test_gemm_attn_gpu import LAYOUTS, gemm_case, qkv_case

pytestmark = pytest.mark.gpu

INSTANCES = [(epi, layout) for epi, layouts in LAYOUTS.items() for layout in layouts]


@pytest.fixture(scope='module')
def ops():
    from diffusion_pipe_b200 import ops as o
    return o


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize('ints', [True, False])
@pytest.mark.parametrize('accumulate', [False, True])
@pytest.mark.parametrize('inst', INSTANCES, ids=[f'{e}-{a}{b}' for e, (a, b) in INSTANCES])
def test_gemm_several_tiles_per_cta(inst, accumulate, ints, ops):
    """2053 x 4136 (17 x 17 tiles, up to 3 per CTA): the last tile has a 5-row M tail and, for STORE, a 40-column N tail
    (one partial 32-column group); fused epilogues take N % 32 == 0 tails of 32 and 96 columns"""
    epi, layout = inst
    M = 2053
    assert -(-M // 128) * 17 > 2 * _sms()
    for n_tail in ((40, 8) if epi == 'store' else (32, 96)):
        gemm_case(ops, M, 16 * 256 + n_tail, 320, epi, layout, bias=epi != 'store' or n_tail == 40,
                  accumulate=accumulate, rpb=M // 3 if epi == 'gate_res' else None, ints=ints, twice=True)


@pytest.mark.parametrize('inst', INSTANCES, ids=[f'{e}-{a}{b}' for e, (a, b) in INSTANCES])
def test_gemm_fewer_tiles_than_sms(inst, ops):
    """12 tiles: most SMs get none, each CTA one tile with a long K"""
    epi, layout = inst
    gemm_case(ops, 385, 776 if epi == 'store' else 800, 2048, epi, layout, accumulate=epi == 'store', twice=True)


@pytest.mark.parametrize('ints', [True, False])
@pytest.mark.parametrize('mlp', [0, 288])
def test_gemm_qkv_rope_several_tiles_per_cta(mlp, ints, ops):
    """24 heads at 2 x 300 rows (5 x 36 QKV tiles, and the MLP half of the fused linear1 with a 32-column N tail): each
    CTA normalises heads of several tiles; a sample boundary and the M tail fall inside tiles"""
    qkv_case(ops, 2, 300, 24, mlp, 7, True, K=192, ints=ints, twice=True)
