"""CPU checks of the ADMM posterior's entry points: they are exported and bound, and without a CUDA device score_var fails loudly
(no CPU fallback).  mlease_admm_posterior needs a session, which cannot be created without a device: that refusal is what is checked
for it here."""
import numpy as np
import pytest


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


@pytest.mark.skipif(_has_gpu(), reason="checks the no-GPU failure mode")
def test_no_cpu_fallback():
    import mlease_b200 as mb
    with pytest.raises(mb.MleaseError, match="no CPU fallback"):
        mb.score_var([0, 1], [0], [1.0], np.zeros(3), var=np.ones(3))
    with pytest.raises(mb.MleaseError, match="no CPU fallback"):
        mb.World([0], 2, 10, [1.0])


def test_entry_points_are_declared_and_bound():
    import mlease_b200 as mb
    from mlease_b200._native import EXPORTED
    for name in ("mlease_admm_posterior", "mlease_world_admm_posterior", "mlease_score_var"):
        assert name in EXPORTED
        assert getattr(mb.lib(), name).restype is not None
