"""HashMatrixTable without a GPU: the host backend refuses it with a clear error (its index is a GPU hash table)."""
import pytest
import torch


def test_host_backend_refuses_hash_table():
    if torch.cuda.is_available():
        pytest.skip("the host backend is chosen only without a CUDA device")
    import multiverso_b200 as mv
    mv.FLAGS.reset()
    mv.init()
    try:
        with pytest.raises(NotImplementedError, match="device backend"):
            mv.HashMatrixTable(10, 4)
    finally:
        mv.shutdown()
        mv.FLAGS.reset()
