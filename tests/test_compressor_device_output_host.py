"""compressobj(..., device_output=True) without a device is refused before the library is called."""
import pytest

import zopfli_b200 as zb


class _NoLibrary:
    """a Library whose every use fails: the refusal must come first"""

    def __getattr__(self, name):
        raise AssertionError("the library was called: %s" % name)


def test_device_output_needs_a_device():
    with pytest.raises(ValueError, match="device_output"):
        zb.Compressor(_NoLibrary(), 0, device_output=True)
    with pytest.raises(ValueError, match="device_output"):
        zb.Library.compressobj(_NoLibrary(), 1, device_output=True)
