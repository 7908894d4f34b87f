"""The 2 GiB guard of concat()'s Utf8 result (string_funcs.cu's render_strings through varlen.cu).

concat(s, <1 MiB literal>) over rows whose s is empty but for the last row.  The result's byte total is known by
construction: rows x 2^20 + |s of the last row|.  A total of exactly 2^31 - 1 fits the int32 offsets and is checked byte
for byte on the device; 2^31 fails with Process "offset overflow", and so does 4097 x 2^20 = 2^32 + 2^20, which an int32
scan wraps back to a positive 2^20.  The exact 64-bit sum comes from concat_lengths_kernel, so protobuf_sum64_kernel never
runs.
"""
import string

import pyarrow as pa
import pytest

from arkflow_b200.arrow_ffi import DeviceBatch
from arkflow_b200.processor import ArkError, SqlProcessor
from test_inputs_edges_gpu import launches

pytestmark = pytest.mark.gpu

MIB = 1 << 20
LITERAL = (string.ascii_letters * (MIB // len(string.ascii_letters) + 1))[:MIB]
QUERY = "SELECT concat(s, '" + LITERAL + "') AS c FROM flow"


@pytest.fixture(scope="module")
def timing(gpu):
    gpu.ark_kernel_timing_enable(1)
    yield gpu
    gpu.ark_kernel_timing_enable(0)


def rows(n, last_len):
    return pa.record_batch({"s": pa.array([""] * (n - 1) + ["z" * last_len], pa.string())})


def test_result_of_2gib_minus_one_bytes(timing):
    import torch

    n = 2047
    timing.ark_kernel_timing_reset()
    out = SqlProcessor({"query": QUERY}).process_device(DeviceBatch.from_arrow(rows(n, MIB - 1)))
    assert (launches(timing, "concat_lengths_kernel"), launches(timing, "protobuf_sum64_kernel")) == (1, 0)
    c = out.columns[0]
    assert out.num_rows == n
    offs = c.offsets.to(torch.int64)
    assert torch.equal(offs[:n], torch.arange(n, device=offs.device, dtype=torch.int64) * MIB)
    assert int(offs[n]) == 2 ** 31 - 1
    got = c.data.tensor()
    assert got.numel() == 2 ** 31 - 1
    lit = torch.frombuffer(bytearray(LITERAL.encode()), dtype=torch.uint8).to(got.device)
    assert bool((got[:(n - 1) * MIB].view(n - 1, MIB) == lit).all())
    last = got[(n - 1) * MIB:]
    assert bool((last[:MIB - 1] == ord("z")).all()) and torch.equal(last[MIB - 1:], lit)
    del got, last
    out.close()


@pytest.mark.parametrize("n, last_len", [(2047, MIB), (4097, 0)], ids=["pow31", "wrap"])
def test_result_past_2gib_is_a_process_error(timing, n, last_len):
    total = n * MIB + last_len
    assert total > 2 ** 31 - 1
    if n == 4097:
        assert 0 < total % 2 ** 32 < 2 ** 31  # the int32 total would look valid
    timing.ark_kernel_timing_reset()
    with pytest.raises(ArkError) as e:
        SqlProcessor({"query": QUERY}).process_device(DeviceBatch.from_arrow(rows(n, last_len)))
    assert e.value.kind == "Process" and "offset overflow" in e.value.message, e.value.message
    assert launches(timing, "protobuf_sum64_kernel") == 0
