"""tools/measure.py, the benchmark scripts' shared helpers: ptxas's report is read without a GPU, and the helpers that
time or read the card refuse to run without one instead of reporting a number that was not measured."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tools'))
import measure  # noqa: E402


def test_ptxas_reports_select_kernels():
    res = measure.ptxas('select.cu', ('k_fov', 'k_sl_'))
    assert res['k_fov']['registers'] > 0
    sl = [k for k in res if k.startswith('k_sl_')]
    assert sl and all(res[k]['registers'] > 0 and res[k]['spill_bytes'] >= 0 for k in sl)
    assert all(k.startswith(('k_fov', 'k_sl_')) for k in res)


@pytest.mark.parametrize('call', [lambda: measure.card(), lambda: measure.time_calls(lambda: None, 1, 0)],
                         ids=['card', 'time_calls'])
def test_gpu_helpers_raise_without_cuda(monkeypatch, call):
    monkeypatch.setattr(torch.cuda, 'is_available', lambda: False)
    with pytest.raises(RuntimeError, match='no CUDA device'):
        call()
