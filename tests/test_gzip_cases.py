"""CPU checks of gzip_cases: every clean stream inflates to its data with zlib, the false-start stream hides a dynamic
block header in a stored block, every refusal is refused, truncated or read on from by zlib, and without a device the
stream layer (the host continuation from the first byte) still reads each of these files exactly as gzread does, in
calls of up to 2^32 + 2 MiB."""
import gzip
import json
import os
import struct
import subprocess
import sys
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


# One call of 2^32 + 2 MiB through the host continuation (a pipe) and through gzread (the regular file): sha256, length,
# error and truncation flag of each. The hook's buffer of that size is not touched beyond the bytes read.
_BIG_READ = r"""
import hashlib, json, sys, threading
import bgzf_cases as B
from ngmlr_b200 import _lib
path, fifo = sys.argv[1:3]
size, cap = (1 << 32) + (2 << 20), 64 << 20
lib = _lib.load()
def feed():
    with open(fifo, "wb") as f:
        f.write(open(path, "rb").read())
t = threading.Thread(target=feed)
t.start()
got = B.stream_read(lib, fifo, B.HOST, size, cap=cap)
t.join()
want = B.stream_read(lib, path, B.GZREAD, size, cap=cap)
print(json.dumps([[hashlib.sha256(r[0]).hexdigest(), len(r[0]), r[1], r[2]] for r in (got, want)]))
"""


def test_host_continuation_reads_4_gib_and_more_in_one_call(tmp_path):
    """zlib takes at most UINT_MAX bytes of output per inflate pass, so a request of 2^32 bytes or more is handed over
    in passes no larger (run in a subprocess with a timeout, so that a read that never returns fails the test)."""
    data = G.fastq(9 << 20)
    path, fifo = str(tmp_path / "big.fq.gz"), str(tmp_path / "pipe")
    with open(path, "wb") as f:
        f.write(G.gz(data))
    os.mkfifo(fifo)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([root, os.path.join(root, "tests")]))
    r = subprocess.run([sys.executable, "-c", _BIG_READ, path, fifo], env=env, capture_output=True, text=True,
                       timeout=300)
    assert r.returncode == 0, r.stderr
    got, want = json.loads(r.stdout)
    assert got == want and want[1] == len(data), (got, want)
