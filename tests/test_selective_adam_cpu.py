"""Refusals of the selective optimiser step that need no GPU: the C layer checks a row mask's row length before any
launch, and FusedAdam.step checks the mask's dtype, device and shape before it touches any state."""
import pytest
import torch

from relightable3dgaussian_b200 import _lib
from relightable3dgaussian_b200.optim import FusedAdam

FAKE = 0x10000      # never dereferenced: every call below is refused before anything is enqueued


def _tensor(n, row_mask, row_elems):
    t = (_lib.AdamTensor * 1)()
    t[0].param = t[0].grad = t[0].exp_avg = t[0].exp_avg_sq = FAKE
    t[0].n, t[0].step, t[0].lr, t[0].beta1, t[0].beta2, t[0].eps = n, 1, 1e-3, 0.9, 0.999, 1e-15
    t[0].row_mask, t[0].row_elems = row_mask, row_elems
    return t


def test_c_layer_refuses_bad_row_lengths():
    lib = _lib.load()
    assert lib.r3dg_adam_step(1, _tensor(12, FAKE, 0), None) == -10001        # row_elems < 1
    assert lib.r3dg_adam_step(1, _tensor(12, FAKE, -3), None) == -10001
    assert lib.r3dg_adam_step(1, _tensor(12, FAKE, 5), None) == -10001        # n not a multiple of row_elems
    assert lib.r3dg_adam_step(1, _tensor(2 << 31, FAKE, 1 << 31), None) == -10002   # rows longer than INT_MAX
    assert lib.r3dg_adam_step(1, _tensor(0, FAKE, 3), None) == 0              # empty tensor: nothing launched
    t = _tensor(0, None, 0)                                                   # no mask: row_elems is not read
    assert lib.r3dg_adam_step(1, t, None) == 0
    assert _lib.AdamTensor().row_mask is None and _lib.AdamTensor().row_elems == 0


def test_step_refuses_bad_masks_before_any_state_change():
    p = torch.zeros(10, 3, requires_grad=True)
    opt = FusedAdam([{"params": [p], "lr": 1e-3, "name": "xyz"}], lr=0.0, eps=1e-15)
    for bad in (torch.ones(10, dtype=torch.bool),                 # CPU
                torch.ones(10),                                   # float
                torch.ones(10, dtype=torch.int32),
                [True] * 10):
        with pytest.raises(ValueError):
            opt.step(visibility=bad)
    assert len(opt.state) == 0
    p.grad = torch.ones(10, 3)                                    # CPU parameter: no fallback, mask or not
    with pytest.raises(RuntimeError):
        opt.step(visibility=torch.ones(10, dtype=torch.bool))
    assert len(opt.state) == 0
