"""GPU: launch_plan.capture_graph, the one place the launch plans and the fused denoising step record their CUDA graphs, pauses
Python's cyclic garbage collector while the stream captures and restores it afterwards.  A launch plan is a reference cycle,
so a dropped plan's CUDA graph is destroyed by the collector, and that destruction must not land inside another capture."""
import gc

import pytest
import torch

pytestmark = pytest.mark.gpu


def test_capture_pauses_the_collector_and_restores_it():
    from kandinsky2.launch_plan import capture_graph
    x = torch.zeros(4, device="cuda")
    seen = []

    def launch():
        seen.append(gc.isenabled())
        x.add_(1.0)

    assert gc.isenabled()
    g = capture_graph(launch)
    assert seen == [False] and gc.isenabled()
    g.replay()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(x, torch.full((4,), 2.0, device="cuda"))
    gc.disable()                      # a caller that had paused it keeps it paused
    try:
        capture_graph(launch)
        assert seen == [False, False] and not gc.isenabled()
    finally:
        gc.enable()


@pytest.mark.filterwarnings("ignore:The CUDA Graph is empty")
def test_a_failed_capture_restores_the_collector():
    from kandinsky2.launch_plan import capture_graph

    def launch():
        raise RuntimeError("launch refused before any work")

    with pytest.raises(RuntimeError, match="launch refused"):
        capture_graph(launch)
    assert gc.isenabled()
    torch.cuda.synchronize()
