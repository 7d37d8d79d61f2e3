"""CPU: what GaussianTrainer.result() does when the last pass overflowed the binning arena, driven through a stub library: which call it
repeats and with which arguments, the step / iteration counters it leaves, and the errors it raises."""
import types

import pytest
import torch

from photo_slam_b200 import _lib
from test_pixel_grads_cpu import _cpu_trainer

RETRY = -4
QUEUED = "queued call\\(s\\) \\(first: pass 1 of 3\\) overflowed the binning arena and were dropped"
PIXELS = "the render that backwardPixels back-propagated through overflowed the binning arena, so that call was a no-op"


class _StubLib:
    """Records every enqueuing call; psb_trainer_result_depth returns the scripted codes, then 0."""

    def __init__(self):
        self.calls, self.results = [], []

    def psb_trainer_forward(self, h, P, M, model, cam, bg, D, out, radii, out_depth, out_alpha, pass_no, stream):
        self.calls.append(("forward", out, radii, out_depth, out_alpha))
        pass_no._obj.value = len(self.calls)
        return 0

    def psb_trainer_step_exposure(self, h, P, M, model, cam, bg, gt, mask, step, out_color, radii, depth, exposure, stream):
        self.calls.append(("step", gt, mask, step._obj.step, step._obj.update_densify_stats, depth is not None, exposure is not None))
        return 0

    def psb_trainer_backward_pixels(self, h, pass_no, P, M, model, cam, bg, px, step, grads, stream):
        self.calls.append(("pixels", pass_no, step._obj.step, grads is None))
        return 0

    def psb_trainer_result_depth(self, h, out, n, stream):
        rc = self.results.pop(0) if self.results else 0
        if rc == 0:
            out[0], out[1], out[2], out[3] = 0.5, 0.25, 0.75, 0.125
            n._obj.value = 7
        return rc


@pytest.fixture
def stubbed(monkeypatch):
    """A trainer whose library is the stub; overflow_info(first, count, current) sets what psb_trainer_overflow_info reports."""
    monkeypatch.setattr(torch.cuda, "current_stream", lambda: types.SimpleNamespace(cuda_stream=None))
    tr, m, cam = _cpu_trainer()
    real, stub = tr.L, _StubLib()
    tr.L = stub
    info = {}
    tr._overflow_info = lambda: info["v"]

    def overflow(first, count, current):
        info["v"] = (first, count, current)
        stub.results = [RETRY]
    yield tr, m, cam, stub, overflow
    tr.L = real


def test_a_render_is_rendered_again(stubbed):
    tr, m, cam, stub, overflow = stubbed
    out, radii = torch.empty((3, cam["H"], cam["W"])), torch.empty(m.num_points(), dtype=torch.int32)
    tr.render(cam, out, radii, check=False)
    overflow(1, 1, 1)
    assert tr.result() == (0.5, 0.25, 0.75, 7)
    assert stub.calls == [("forward", out.data_ptr(), radii.data_ptr(), None, None)] * 2
    assert (m.step_, tr.iteration) == (0, 0)


@pytest.mark.parametrize("with_depth", [False, True], ids=["result", "result_depth"])
def test_a_step_is_rolled_back_and_repeated(stubbed, with_depth):
    tr, m, cam, stub, overflow = stubbed
    gt, gd = torch.zeros((3, cam["H"], cam["W"])), torch.ones((cam["H"], cam["W"]))
    tr.trainForOneIteration(cam, gt, gt_depth=gd, lambda_depth=0.1, exposure_id=0, densify_stats=False)
    overflow(1, 1, 1)
    res = tr.result_depth() if with_depth else tr.result()
    assert res == ((0.5, 0.25, 0.75, 0.125, 7) if with_depth else (0.5, 0.25, 0.75, 7))
    assert stub.calls == [("step", gt.data_ptr(), None, 1, 0, True, True)] * 2   # the same step number: the first was undone
    assert (m.step_, tr.iteration) == (1, 1)


def test_train_with_loss_is_rolled_back_and_repeated(stubbed):
    tr, m, cam, stub, overflow = stubbed
    seen = []

    def loss_fn(image, depth):   # (the stub renders nothing: the loss counts the calls)
        seen.append(image.shape)
        return torch.nan_to_num(image).mul(0).sum() + torch.nan_to_num(depth).mul(0).sum() + len(seen)
    assert float(tr.trainWithLoss(cam, loss_fn, depth=True)) == 1.0
    overflow(1, 1, 1)
    res = tr.result()
    assert res[0] == 2.0 and all(x != x for x in res[1:3]) and res[3] == 7   # the repeated call's loss
    assert [c[0] for c in stub.calls] == ["forward", "pixels"] * 2 and len(seen) == 2
    assert stub.calls[1][2] == stub.calls[3][2] == 1 and stub.calls[1][3] and stub.calls[3][3]   # the same Adam step, twice
    assert (m.step_, tr.iteration) == (1, 1)
    assert all(x != x for x in tr.result_depth()[1:4])


@pytest.mark.parametrize("adam", [True, False], ids=["adam", "grads"])
def test_backward_pixels_is_not_repeated(stubbed, adam):
    tr, m, cam, stub, overflow = stubbed
    tr.render(cam, check=False)
    grads = None if adam else [torch.zeros_like(t) for t in m.tensors()]
    tr.backwardPixels(torch.zeros((3, cam["H"], cam["W"])), grads=grads)
    assert (m.step_, tr.iteration) == ((1, 1) if adam else (0, 0))
    overflow(1, 1, 1)
    with pytest.raises(_lib.PsbError, match=PIXELS):
        tr.result()
    assert [c[0] for c in stub.calls] == ["forward", "pixels"]
    assert (m.step_, tr.iteration) == (0, 0)
    assert tr.result() == (0.5, 0.25, 0.75, 7)


@pytest.mark.parametrize("last", ["step", "train_with_loss", "pixels_adam", "render", "pixels_grads"])
def test_a_queued_overflow_rolls_back_count_steps_when_the_last_call_advanced(stubbed, last):
    tr, m, cam, stub, overflow = stubbed
    gt = torch.zeros((3, cam["H"], cam["W"]))
    tr.trainForOneIteration(cam, gt)
    tr.trainForOneIteration(cam, gt)
    if last == "step":
        tr.trainForOneIteration(cam, gt)
    elif last == "train_with_loss":
        tr.trainWithLoss(cam, lambda image: image.sum())
    elif last == "render":
        tr.render(cam, check=False)
    else:
        tr.render(cam, check=False)
        tr.backwardPixels(torch.zeros((3, cam["H"], cam["W"])), grads=None if last == "pixels_adam" else [torch.zeros_like(t) for t in m.tensors()])
    before, calls = (m.step_, tr.iteration), len(stub.calls)
    overflow(1, 3, 3)
    with pytest.raises(_lib.PsbError, match=QUEUED):
        tr.result()
    advanced = last in ("step", "train_with_loss", "pixels_adam")
    assert (m.step_, tr.iteration) == ((before[0] - 3, before[1] - 3) if advanced else before)
    assert len(stub.calls) == calls   # nothing repeated


def test_a_single_overflow_of_an_earlier_pass_is_a_queued_overflow(stubbed):
    tr, m, cam, stub, overflow = stubbed
    gt = torch.zeros((3, cam["H"], cam["W"]))
    tr.trainForOneIteration(cam, gt)
    tr.trainForOneIteration(cam, gt)
    overflow(1, 1, 2)
    with pytest.raises(_lib.PsbError, match="1 queued call\\(s\\) \\(first: pass 1 of 2\\)"):
        tr.result()
    assert (m.step_, tr.iteration) == (1, 1) and len(stub.calls) == 2
