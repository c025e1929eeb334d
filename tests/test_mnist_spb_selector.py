"""``choose_spb``, the samples per CTA of the fp32 batch-split training kernel, as a plain function."""
from nn_distributed_training_b200.ops.mnist_fused import choose_spb


def test_choose_spb_at_batch_100_on_132_sms():
    """The samples per CTA the solo and individual-training runs (batch 100) get on an H100 SXM: the smallest count
    whose L x ceil(100 / spb) CTAs fit in one wave of 132 SMs; 10 nodes is the paper's graph.  Each of 4..8 is one
    instantiation that tests/test_gpu_mnist_batch_split.py runs."""
    assert [choose_spb(100, L, 132) for L in (3, 6, 7, 8, 10)] == [4, 5, 6, 7, 8]
    assert choose_spb(100, 20, 132) == 8            # no count fits one wave: the largest
