"""The stream group's step sizes (include/w2l.h w2l_stream_group_buckets, host code, no GPU): a tick's pooled rows run as
full max_batch steps, then the rest in the smallest power-of-two bucket (or max_batch) that holds it."""
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from wav2lip_b200 import _lib, stream  # noqa: E402


def _expected(max_batch, n):
    out = [max_batch] * (n // max_batch)
    rest = n % max_batch
    if rest:
        b = 1
        while b < rest:
            b *= 2
        out.append(min(b, max_batch))
    return out


@pytest.mark.parametrize("max_batch", [1, 2, 3, 4, 16, 100, 128])
def test_buckets(max_batch):
    for n in list(range(0, 3 * max_batch + 2)) + [1000, 4097]:
        got = stream.stream_buckets(max_batch, n)
        assert got == _expected(max_batch, n), (max_batch, n)
        assert sum(got) >= n and all(b <= max_batch for b in got)
        # padding stays below half a bucket, except for buckets of 1 and max_batch
        if got and got[-1] not in (1, max_batch):
            assert n - max_batch * (len(got) - 1) > got[-1] // 2


def test_bucket_sizes_are_few():
    """A group of max_batch 128 pins at most these eight plans whatever its traffic."""
    sizes = set()
    for n in range(0, 600):
        sizes.update(stream.stream_buckets(128, n))
    assert sizes == {1, 2, 4, 8, 16, 32, 64, 128}
    assert set().union(*[stream.stream_buckets(100, n) for n in range(300)]) == {1, 2, 4, 8, 16, 32, 64, 100}


def test_bad_arguments():
    with pytest.raises(_lib.W2LError):
        stream.stream_buckets(0, 5)
    with pytest.raises(_lib.W2LError):
        stream.stream_buckets(4, -1)
