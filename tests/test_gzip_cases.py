"""CPU checks of gzip_cases: every clean stream inflates to its data with zlib, the false-start stream hides a dynamic
block header in a stored block, every refusal is refused, truncated or read on from by zlib, and without a device the
stream layer still reads each of these files exactly as gzread does."""
import gzip
import struct
import zlib

import pytest

import bgzf_cases as B
import gzip_cases as G
from ngmlr_b200 import _lib


@pytest.fixture(scope="module")
def clean():
    return G.clean()


def test_clean_streams_inflate_to_their_data(clean):
    for name, (blob, data) in clean.items():
        assert gzip.decompress(blob) == data, name
    assert len(B.members(clean["300_members"][0])) == 0  # plain gzip, not BGZF
    blob = clean["false_start"][0]
    assert blob[10] == 0  # a non-final stored block first
    n = struct.unpack_from("<H", blob, 11)[0]
    payload = blob[15:15 + n]
    assert (payload[0] >> 1) & 3 == 2  # its payload starts with a dynamic block header


def test_refusals_are_not_clean():
    for name, blob in G.refusals().items():
        d = zlib.decompressobj(31)
        try:
            out = d.decompress(blob)
            bad = not d.eof or d.unused_data != b""
        except zlib.error:
            bad = True
        assert bad, name


@pytest.mark.parametrize("size", [4096, 3 << 20])
def test_stream_layer_without_device_equals_gzread(tmp_path, clean, size):
    lib = _lib.load()
    files = {k: v[0] for k, v in clean.items() if len(v[1]) < 8 << 20}
    files.update(G.refusals())
    for name, blob in files.items():
        path = str(tmp_path / (name + ".gz"))
        with open(path, "wb") as f:
            f.write(blob)
        want = B.stream_read(lib, path, B.GZREAD, size, cap=64 << 20)
        got = B.stream_read(lib, path, B.HOST, size, cap=64 << 20)
        assert got[:3] == want[:3], name
