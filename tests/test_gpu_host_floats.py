"""GPU: the tracer's host copy of the camera centre (ops._host_floats) never returns the values of an earlier tensor
that the caching allocator placed at the same address."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def test_new_tensor_at_a_freed_address_reads_its_own_values(cuda_dev):
    from selfreconcode_b200 import ops
    ops._host_cache.clear()
    for i in range(80):                     # more than the cache holds: entries are dropped and addresses recycled
        cam = torch.tensor([float(i), 0.5, 2.5], device=cuda_dev)
        assert ops._host_floats(cam) == (float(i), 0.5, 2.5)
        del cam
    cam = torch.tensor([1.0, 2.0, 3.0], device=cuda_dev)
    assert ops._host_floats(cam) == (1.0, 2.0, 3.0)
    cam.add_(1.0)                           # in place: a new version, read again
    assert ops._host_floats(cam) == (2.0, 3.0, 4.0)
