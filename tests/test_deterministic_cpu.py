"""CPU: the deterministic-mode switch of the trainer context — declared, exported, validated before any CUDA call, and followed by
the Python trainers' deterministic=None."""
import os

import pytest
import torch

from photo_slam_b200 import _lib

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "psb200.h")


def test_symbol_declared_and_exported():
    assert "psb_trainer_set_deterministic" in _lib.exported_symbols()
    assert "int psb_trainer_set_deterministic(psb_trainer* t, int enable);" in open(HEADER).read()
    assert hasattr(_lib.lib(), "psb_trainer_set_deterministic")


def test_null_context_is_an_argument_error():
    from photo_slam_b200 import trainer
    L = trainer._bind()
    assert L.psb_trainer_set_deterministic(None, 1) == -1
    assert L.psb_trainer_set_deterministic(None, 0) == -1


@pytest.fixture
def torch_deterministic_flag():
    before, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    yield
    torch.use_deterministic_algorithms(before, warn_only=warn)


def test_python_default_follows_the_torch_flag(torch_deterministic_flag):
    """deterministic=None follows torch.use_deterministic_algorithms at each training call; True / False force the mode. Setting the
    mode needs no device (the context makes its scratch at the next pass)."""
    from photo_slam_b200 import trainer
    model = trainer.GaussianModel(device="cpu")
    follow = trainer.GaussianTrainer(model, background=torch.zeros(3))
    on = trainer.GaussianTrainer(model, background=torch.zeros(3), deterministic=True)
    off = trainer.GaussianTrainer(model, background=torch.zeros(3), deterministic=False)
    assert on._det_applied and not off._det_applied

    torch.use_deterministic_algorithms(True)
    assert follow.deterministic and on.deterministic and not off.deterministic
    follow._apply_deterministic()
    assert follow._det_applied
    torch.use_deterministic_algorithms(False)
    assert not follow.deterministic and on.deterministic and not off.deterministic
    follow._apply_deterministic()
    assert not follow._det_applied
