"""The `file` input reports a missing path from connect() for every format before it touches a device, so the message is
the same with or without a GPU: Process "Read input failed: Object at location <path> not found"."""
import pytest

from arkflow_b200.input import FileInput
from arkflow_b200.processor import ArkError


@pytest.mark.parametrize("fmt", ["csv", "json", "avro", "arrow"])
def test_missing_path_needs_no_device(tmp_path, fmt):
    p = tmp_path / f"missing.{fmt}"
    inp = FileInput({"input_type": {"type": fmt, "path": str(p)}})
    with pytest.raises(ArkError) as e:
        inp.connect()
    assert (e.value.kind, e.value.message) == ("Process", f"Read input failed: Object at location {p} not found")
