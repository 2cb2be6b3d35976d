"""Read loading speed: ngmlr_b200_reads_load (B200Aligner.load_reads) on a synthetic FASTQ shaped like bench.py's
pacbio50 reads (lognormal lengths, median 8 000, at most 40 000 bases; 4-line records, Phred+33 qualities), plain and
gzip, next to the unmodified ReadProvider on one thread (ref_read_file of oracle/_ref/libngmlr_reads.so, where built).

Reports GB/s of stream text and Gbp/s of bases for each, the host read / inflate, device parse and gather phases, and
the peak device memory of the run (cudaMemGetInfo sampled after every batch, less the level before the first load).
Prints one JSON object, and writes it to --out where given.

    python scripts/read_load_timing.py --gb 4 [--gzip-gb 1] [--oracle-gb 0.5]"""
import argparse
import ctypes as C
import gzip
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def write_fastq(path, gb, seed=1, opener=open):
    rng = np.random.default_rng(seed)
    acgt = np.frombuffer(b"ACGT", dtype=np.uint8)
    target, written, bases, i = int(gb * 1e9), 0, 0, 0
    with opener(path, "wb") as f:
        while written < target:
            lens = np.clip(rng.lognormal(np.log(8000), 0.6, 512).astype(np.int64), 200, 40000)
            seq = acgt[rng.integers(0, 4, int(lens.sum()))]
            qual = rng.integers(33, 75, int(lens.sum())).astype(np.uint8)
            parts, o = [], 0
            for L in lens:
                parts.append(b"@m%d/ccs\n%s\n+\n%s\n" % (i, seq[o:o + L].tobytes(), qual[o:o + L].tobytes()))
                o += L
                i += 1
            blob = b"".join(parts)
            f.write(blob)
            written += len(blob)
            bases += int(lens.sum())
    return written, bases, i


def free_bytes():
    import torch
    free, _ = torch.cuda.mem_get_info(0)
    return free


def time_loader(path, stream_bytes, bases, chunk_bytes, max_bases):
    from ngmlr_b200 import B200Aligner
    a = B200Aligner(0)
    base_free = free_bytes()
    low = base_free
    n = 0
    t0 = time.perf_counter()
    for batch in a.load_reads(path, max_reads=1_000_000, max_bases=max_bases, chunk_bytes=chunk_bytes):
        n += len(batch.reads)
        low = min(low, free_bytes())
    dt = time.perf_counter() - t0
    a.close()
    return dict(seconds=dt, reads=n, gb_per_s=stream_bytes / dt / 1e9, gbp_per_s=bases / dt / 1e9,
                peak_device_bytes=base_free - low)


def time_native(path, chunk_bytes, max_bases):
    """The C ABI alone (no Python record objects): load calls back to back, with the handle's phase times."""
    from ngmlr_b200 import B200Aligner, _lib
    from ngmlr_b200.samtext import SamRead
    a = B200Aligner(0)
    lib = a.lib
    f = C.c_void_p()
    assert lib.ngmlr_b200_read_file_open(path.encode(), C.byref(_lib.ReadFileOptions(chunk_bytes)), C.byref(f)) == 0
    recs = (SamRead * 200_000)()
    nr, nd = C.c_int32(0), C.c_int32(0)
    t0 = time.perf_counter()
    total = 0
    while True:
        a._check(lib.ngmlr_b200_reads_load(a.h, f, 200_000, max_bases, 256, recs, C.byref(nr), C.byref(nd)))
        if nr.value == 0:
            break
        total += nr.value
    dt = time.perf_counter() - t0
    sb, rc, dev = C.c_int64(0), C.c_int64(0), C.c_int64(0)
    ms = [C.c_float(0) for _ in range(3)]
    lib.ngmlr_b200_read_file_stats(f, C.byref(sb), C.byref(rc), C.byref(ms[0]), C.byref(ms[1]), C.byref(ms[2]),
                                   C.byref(dev))
    lib.ngmlr_b200_read_file_close(f)
    a.close()
    return dict(seconds=dt, reads=total, gb_per_s=sb.value / dt / 1e9, read_ms=ms[0].value, parse_ms=ms[1].value,
                gather_ms=ms[2].value, handle_device_bytes=dev.value)


def time_oracle(path, stream_bytes, bases):
    full = os.path.join(ROOT, "oracle", "_ref", "libngmlr_reads.so")
    if not os.path.exists(full):
        return None
    import read_loader_cases as R
    t0 = time.perf_counter()
    out = path + ".oracle"
    r = subprocess.run([sys.executable, "-c", R._SCRIPT, full, path, "256", out], capture_output=True, timeout=7200)
    dt = time.perf_counter() - t0
    os.unlink(out)
    return dict(seconds=dt, returncode=r.returncode, gb_per_s=stream_bytes / dt / 1e9, gbp_per_s=bases / dt / 1e9,
                note="includes writing every read to a file and the start of a Python process")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gb", type=float, default=4.0, help="plain FASTQ size")
    ap.add_argument("--gzip-gb", type=float, default=1.0, help="FASTQ size (uncompressed) of the gzip run")
    ap.add_argument("--oracle-gb", type=float, default=0.5, help="FASTQ size of the ReadProvider run")
    ap.add_argument("--chunk-mb", type=int, default=256)
    ap.add_argument("--max-bases", type=int, default=200_000_000)
    ap.add_argument("--dir", default=None)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    props = torch.cuda.get_device_properties(0)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    d = args.dir or tempfile.mkdtemp(prefix="read_load_")
    res = dict(gpu=props.name, nvidia_smi=smi.stdout.strip(), chunk_mb=args.chunk_mb)
    plain = os.path.join(d, "reads.fq")
    sb, bases, n = write_fastq(plain, args.gb)
    res["plain_file"] = dict(bytes=sb, bases=bases, reads=n)
    chunk = args.chunk_mb << 20
    time_loader(plain, sb, bases, chunk, args.max_bases)  # page cache and module load
    res["plain"] = time_loader(plain, sb, bases, chunk, args.max_bases)
    res["plain_native"] = time_native(plain, chunk, args.max_bases)
    os.unlink(plain)
    gz = os.path.join(d, "reads.fq.gz")
    gsb, gbases, _ = write_fastq(gz, args.gzip_gb, seed=2, opener=lambda p, m: gzip.open(p, m, compresslevel=1))
    res["gzip"] = time_loader(gz, gsb, gbases, chunk, args.max_bases)
    res["gzip"]["compressed_bytes"] = os.path.getsize(gz)
    os.unlink(gz)
    if args.oracle_gb > 0:
        small = os.path.join(d, "small.fq")
        osb, obases, _ = write_fastq(small, args.oracle_gb, seed=3)
        res["readprovider_one_thread"] = time_oracle(small, osb, obases)
        res["readprovider_loader_same_file"] = time_loader(small, osb, obases, chunk, args.max_bases)
        os.unlink(small)
    print(json.dumps(res, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
