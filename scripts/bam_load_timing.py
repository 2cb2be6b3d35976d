"""BAM loading speed: ngmlr_b200_reads_load through the C ABI on the same reads written as BGZF BAM and as BGZF FASTQ
(both level 6, compressed by a process pool), shaped like bench.py's pacbio50 reads (lognormal lengths, median 8 000,
at most 40 000 bases, Phred+33 qualities; unaligned records as PacBio writes them), and on SRA-shaped 36 bp reads, the
case with the most records per byte for the host's record walk.

Reports, for each file: GB/s of file, Gbp/s, the host read / inflate, header + record walk (parse_ms) and
upload + decode + copy back (gather_ms) milliseconds, the decode kernels' device time (k_bam_seq, k_bam_qual and
k_bam_subreads, from torch.profiler over one more load), and the BAM load's time over the FASTQ load's, the two
alternated. Prints one JSON object, and writes it to --out where given.

    python scripts/bam_load_timing.py --gb 2 [--short-gb 0.3] [--repeat 3]"""
import argparse
import json
import os
import struct
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))

NT16_CODE = np.zeros(256, dtype=np.uint8)
for _i, _c in enumerate(b"=ACMGRSVTWYHKDBN"):
    NT16_CODE[_c] = _i


def bam_header():
    text = b"@HD\tVN:1.6\tSO:unknown\n@RG\tID:r\tPL:PACBIO\n"
    return b"BAM\1" + struct.pack("<i", len(text)) + text + struct.pack("<i", 0)


def bam_record(name, seq, qual):
    """An unaligned record (flag 4) of ASCII bases and Phred+33 qualities (uint8 arrays)."""
    codes = NT16_CODE[seq]
    if len(codes) % 2:
        codes = np.append(codes, 0)
    packed = (codes[0::2] << 4 | codes[1::2]).astype(np.uint8).tobytes()
    body = struct.pack("<iiBBHHHiiii", -1, -1, len(name) + 1, 255, 4680, 0, 4, len(seq), -1, -1, 0) + name + b"\0" + \
        packed + (qual - 33).tobytes()
    return struct.pack("<i", len(body)) + body


def write_pair(fq_path, bam_path, gb, short, seed=1):
    """The same reads as FASTQ text and as an uncompressed BAM stream; gb of FASTQ text."""
    rng = np.random.default_rng(seed)
    acgt = np.frombuffer(b"ACGT", dtype=np.uint8)
    target, written, bases, i, bam_bytes = int(gb * 1e9), 0, 0, 0, 0
    with open(fq_path, "wb") as fq, open(bam_path, "wb") as bam:
        h = bam_header()
        bam.write(h)
        bam_bytes += len(h)
        while written < target:
            lens = np.full(4096, 36) if short else \
                np.clip(rng.lognormal(np.log(8000), 0.6, 512).astype(np.int64), 200, 40000)
            seq = acgt[rng.integers(0, 4, int(lens.sum()))]
            qual = rng.integers(33, 75, int(lens.sum())).astype(np.uint8)
            fparts, bparts, o = [], [], 0
            for L in lens:
                name = (b"SRR000001.%d" % i) if short else (b"m%d/ccs" % i)
                s, q = seq[o:o + L], qual[o:o + L]
                fparts.append(b"@%s\n%s\n+\n%s\n" % (name, s.tobytes(), q.tobytes()))
                bparts.append(bam_record(name, s, q))
                o += L
                i += 1
            fb, bb = b"".join(fparts), b"".join(bparts)
            fq.write(fb)
            bam.write(bb)
            written += len(fb)
            bam_bytes += len(bb)
            bases += int(lens.sum())
    return dict(fastq_bytes=written, bam_bytes=bam_bytes, bases=bases, reads=i)


def time_native(path, chunk_bytes, max_bases):
    import read_load_timing as RT
    return RT.time_native(path, chunk_bytes, max_bases)


def decode_kernel_ms(path, chunk_bytes, max_bases):
    """Device time of the BAM decode kernels over one load of the file (torch.profiler's CUDA activity)."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        time_native(path, chunk_bytes, max_bases)
    total = {}
    for e in prof.events():
        if "k_bam_" in e.name:
            k = e.name.split("k_bam_")[1].split("(")[0].split("E")[0]
            total["k_bam_" + k] = total.get("k_bam_" + k, 0.0) + e.device_time_total / 1e3
    return total


def bam_counters(path):
    import ctypes as C
    from ngmlr_b200 import B200Aligner, _lib
    from ngmlr_b200.samtext import SamRead
    a = B200Aligner(0)
    lib = a.lib
    f = C.c_void_p()
    assert lib.ngmlr_b200_read_file_open(path.encode(), C.byref(_lib.ReadFileOptions(0)), C.byref(f)) == 0
    recs = (SamRead * 1)()
    nr, nd = C.c_int32(0), C.c_int32(0)
    a._check(lib.ngmlr_b200_reads_load(a.h, f, 1, 0, 256, recs, C.byref(nr), C.byref(nd)))
    st = [C.c_int64(0) for _ in range(5)]
    lib.ngmlr_b200_read_file_bam_stats(f, *[C.byref(x) for x in st])
    fmt = lib.ngmlr_b200_read_file_format(f)
    lib.ngmlr_b200_read_file_close(f)
    a.close()
    return dict(format=fmt, header_bytes=st[0].value)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gb", type=float, default=2.0, help="FASTQ text of the pacbio50-shaped reads")
    ap.add_argument("--short-gb", type=float, default=0.3, help="FASTQ text of the 36 bp reads (0: none)")
    ap.add_argument("--chunk-mb", type=int, default=256)
    ap.add_argument("--max-bases", type=int, default=200_000_000)
    ap.add_argument("--repeat", type=int, default=3, help="loads of each file, alternated")
    ap.add_argument("--dir", default=None)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import bgzf_cases as BG
    props = torch.cuda.get_device_properties(0)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    d = args.dir or tempfile.mkdtemp(prefix="bam_load_")
    res = dict(gpu=props.name, nvidia_smi=smi.stdout.strip(), chunk_mb=args.chunk_mb)
    chunk = args.chunk_mb << 20
    for key, gb, short in (("pacbio50", args.gb, False), ("short36", args.short_gb, True)):
        if gb <= 0:
            continue
        fq, bam = os.path.join(d, key + ".fq"), os.path.join(d, key + ".bam.raw")
        info = write_pair(fq, bam, gb, short)
        fqz, bamz = fq + ".bgz", os.path.join(d, key + ".bam")
        info["fastq_bgzf_bytes"] = BG.compress_file(fq, fqz, 6)
        info["bam_bgzf_bytes"] = BG.compress_file(bam, bamz, 6)
        os.unlink(fq)
        os.unlink(bam)
        info.update(bam_counters(bamz))
        runs = {"fastq": [], "bam": []}
        time_native(fqz, chunk, args.max_bases)  # page cache and module load
        time_native(bamz, chunk, args.max_bases)
        for _ in range(args.repeat):
            runs["fastq"].append(time_native(fqz, chunk, args.max_bases))
            runs["bam"].append(time_native(bamz, chunk, args.max_bases))
        out = dict(files=info)
        for fmt, path in (("fastq", fqz), ("bam", bamz)):
            size = os.path.getsize(path)
            secs = [r["seconds"] for r in runs[fmt]]
            out[fmt] = dict(seconds=secs, file_gb_per_s=[size / s / 1e9 for s in secs],
                            gbp_per_s=[info["bases"] / s / 1e9 for s in secs],
                            read_ms=[r["read_ms"] for r in runs[fmt]], parse_ms=[r["parse_ms"] for r in runs[fmt]],
                            gather_ms=[r["gather_ms"] for r in runs[fmt]],
                            inflate_kernel_ms=[r["inflate_kernel_ms"] for r in runs[fmt]],
                            handle_device_bytes=runs[fmt][-1]["handle_device_bytes"], reads=runs[fmt][-1]["reads"])
        out["bam"]["decode_kernel_ms"] = decode_kernel_ms(bamz, chunk, args.max_bases)
        out["bam_time_over_fastq"] = [b / f for b, f in zip(out["bam"]["seconds"], out["fastq"]["seconds"])]
        res[key] = out
        os.unlink(fqz)
        os.unlink(bamz)
    print(json.dumps(res, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
