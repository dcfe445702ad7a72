"""engine.capture_graphs: every body runs once outside the capture, in order, before each is captured once in the same order; what
`restore` names keeps its value from before the call."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def test_restore_undoes_the_warm_up():
    from diff_pruning_b200.engine import capture_graphs
    acc = torch.full((4,), 5.0, device="cuda")
    log = []

    def body():
        log.append(torch.cuda.is_current_stream_capturing())
        acc.add_(1)
    g, = capture_graphs(acc.device, body, restore=(acc, None))
    torch.cuda.synchronize()
    assert log == [False, True]
    assert torch.equal(acc, torch.full_like(acc, 5.0))
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(acc, torch.full_like(acc, 6.0))


def test_bodies_warm_up_then_capture_in_order():
    from diff_pruning_b200.engine import capture_graphs
    xa, xb = torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda")
    log = []

    def a():
        log.append(("a", torch.cuda.is_current_stream_capturing()))
        xa.add_(1)

    def b():
        log.append(("b", torch.cuda.is_current_stream_capturing()))
        xb.add_(10)
    ga, gb = capture_graphs(xa.device, a, b)
    torch.cuda.synchronize()
    assert log == [("a", False), ("b", False), ("a", True), ("b", True)]
    assert (xa.item(), xb.item()) == (1.0, 10.0)      # nothing restored: the warm-up's updates stay
    ga.replay()
    torch.cuda.synchronize()
    assert (xa.item(), xb.item()) == (2.0, 10.0)
    gb.replay()
    torch.cuda.synchronize()
    assert (xa.item(), xb.item()) == (2.0, 20.0)
