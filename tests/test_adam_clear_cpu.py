"""CPU: b200_adam_update's zero_grad takes 0 (keep), 1 (clear) or B200_ADAM_CLEAR_ON_VETO (clear on a vetoed step only),
the value gsplat.optim passes for FlatAdam.update_state(zero_grad="veto"), and reports any other value before touching
a device."""
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _update(lib, zero_grad):
    from gsplat import _lib

    # numel 0: the arguments are checked, then nothing is launched
    return _lib.check(lib.b200_adam_update(0, 0, None, None, None, None, 0, None, None, None, 0.9, 0.999, 1e-15, 1.0,
                                           zero_grad, 0, None))


def test_clear_on_veto_matches_the_header():
    from gsplat.optim import CLEAR_ON_VETO

    src = open(os.path.join(ROOT, "include", "b200splat.h")).read()
    assert f"#define B200_ADAM_CLEAR_ON_VETO {CLEAR_ON_VETO}\n" in src


def test_zero_grad_values():
    from gsplat import _lib
    from gsplat.optim import CLEAR_ON_VETO

    lib = _lib.load()
    for ok in (0, 1, CLEAR_ON_VETO):
        _update(lib, ok)
    for bad in (-1, CLEAR_ON_VETO + 1):
        with pytest.raises(RuntimeError, match="zero_grad"):
            _update(lib, bad)
