"""Full-size string sort: array_sort_indices over the 500M-row large_utf8 word column of bench.make_word_column (1M
distinct words of 8-16 B, 10 % nulls), both orders.  A word's first five letters are the base-26 digits of its id, most
significant first, and the rest depends on the id only, so the string order is the id order: the expected result is a
stable torch sort of the ids with the nulls moved to the end, compared on the device element for element.

Set B200_FULLSIZE_ROWS to shrink the run (the column has half that many rows; default 1_000_000_000)."""
import os

import pyarrow as pa
import pytest

import arrow_b200.compute as bc
from arrow_b200 import DeviceArray

pytestmark = pytest.mark.gpu
M = int(os.environ.get("B200_FULLSIZE_ROWS", "1000000000")) // 2
SEED = 0x0FF1CE


def test_word_column_sort_fullsize(ctx):
    import gc

    import torch

    from bench import make_validity, make_word_column, unpack_bits
    gc.collect()
    torch.cuda.empty_cache()
    ctx.sync()
    ctx.trim()
    free, _ = torch.cuda.mem_get_info()
    if free < 120 * M:
        pytest.skip(f"needs ~{120 * M >> 30} GiB of free device memory")
    gen = torch.Generator(device="cuda")
    gen.manual_seed(SEED)
    vocab = 1_000_000 if M >= 10_000_000 else max(100, M // 100)
    kid, offs, data, _ = make_word_column(torch, gen, M, vocab)
    valid_bits, nulls = make_validity(torch, M, gen)
    torch.cuda.synchronize()
    words = DeviceArray.from_pointers(ctx, pa.large_string(), M, offs.data_ptr(), validity_ptr=valid_bits.data_ptr(),
                                      null_count=nulls, data2_ptr=data.data_ptr())
    valid = unpack_bits(torch, valid_bits, M)
    for order in ("ascending", "descending"):
        torch.cuda.synchronize()
        got = bc.array_sort_indices(words, order)
        ctx.sync()
        ctx.trim()
        got_t = torch.as_tensor(_Cai(got.buffers[1].ptr, M), device="cuda")
        key = kid if order == "ascending" else (vocab - 1) - kid
        key = torch.where(valid, key, vocab)  # nulls after every word, in row order
        want = torch.sort(key, stable=True).indices
        assert torch.equal(got_t, want), order
        del got_t, got, key, want
        torch.cuda.empty_cache()


class _Cai:
    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<i8", "data": (ptr, False), "version": 2}
