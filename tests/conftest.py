import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (H100); run with `-m gpu` on a GPU machine')


@pytest.fixture(scope='session')
def golden_dir():
    return os.path.join(ROOT, 'tests', 'golden')


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        # a hung kernel must not hold a GPU box until the caller's limit: a watchdog thread ends the process instead
        for item in items:
            if 'gpu' in item.keywords and item.get_closest_marker('timeout') is None:
                item.add_marker(pytest.mark.timeout(900, method='thread'))
        return
    skip = pytest.mark.skip(reason='no CUDA device')
    for item in items:
        if 'gpu' in item.keywords:
            item.add_marker(skip)


@pytest.fixture(autouse=True)
def _poison_uninitialised_cuda_memory(request, monkeypatch):
    """DPIPE_TEST_POISON_EMPTY_CUDA=1 (opt-in, GPU tests): torch.empty / empty_like / new_empty return NaN-filled CUDA
    tensors, so an element that no kernel wrote — a tile tail, a padded row, a skipped output — shows up as NaN instead of
    whatever the caching allocator left there.  The CPU counterpart is always on for the kernel test doubles
    (tests/kernel_doubles.py)."""
    if os.environ.get('DPIPE_TEST_POISON_EMPTY_CUDA', '0') != '1' or 'gpu' not in request.keywords:
        yield
        return
    import torch
    real_empty, real_empty_like, real_new_empty = torch.empty, torch.empty_like, torch.Tensor.new_empty
    skip = (torch.float8_e4m3fn, torch.float8_e5m2)

    def poison(t):
        if torch.is_tensor(t) and t.is_cuda and t.is_floating_point() and t.numel() and t.dtype not in skip:
            t.fill_(float('nan'))
        return t
    monkeypatch.setattr(torch, 'empty', lambda *a, **k: poison(real_empty(*a, **k)))
    monkeypatch.setattr(torch, 'empty_like', lambda *a, **k: poison(real_empty_like(*a, **k)))
    monkeypatch.setattr(torch.Tensor, 'new_empty', lambda self, *a, **k: poison(real_new_empty(self, *a, **k)))
    yield
