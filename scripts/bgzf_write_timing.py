"""BGZF writer speed and ratio: ngmlr_b200_bgzf_* on BAM and SAM text of synthetic mapped reads (the fixture of
tests/test_gpu_bgzf_write.py, repeated to --mb), against host zlib on the same 0xff00 pieces.

Reports, per format: the device deflate rate (input bytes over the CUDA-event time of the device work, copies
excluded), the writer's end-to-end rate into a file in a temporary directory (open to close, wall clock; also from
the first write on, and the open's page-locked and device allocations on their own), the deflate
payload against zlib levels 1 and 6 (raw deflate, one compressobj per piece), zlib's rate at 1 thread and at all
cores (a process pool over the pieces), and the card's name and power limit. Prints one JSON object, and writes it
to --out where given.

    python scripts/bgzf_write_timing.py --mb 512 [--chunk-mb 64] [--repeat 3]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
import zlib
from concurrent.futures import ProcessPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

BLOCK = 0xff00


def _zlib(args):
    piece, level = args
    c = zlib.compressobj(level, zlib.DEFLATED, -15)
    return len(c.compress(piece) + c.flush())


def zlib_pass(pieces, level, workers):
    t = time.perf_counter()
    if workers == 1:
        size = sum(_zlib((p, level)) for p in pieces)
    else:
        with ProcessPoolExecutor(workers) as ex:
            size = sum(ex.map(_zlib, [(p, level) for p in pieces], chunksize=64))
    return size, time.perf_counter() - t


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mb", type=int, default=512)
    ap.add_argument("--chunk-mb", type=int, default=64)
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--zlib-mb", type=int, default=128, help="bytes of each stream zlib compresses (a prefix)")
    ap.add_argument("--out")
    args = ap.parse_args()

    import bam_write_cases as bw
    from ngmlr_b200 import B200Aligner, samtext

    reads, names, lens = bw.mapped_synthetic_reads()
    targets = [b"sim_a", b"sim_b"]
    streams = {"bam": samtext.bam_format(reads, names, targets), "sam": samtext.sam_format(reads, names)}
    a = B200Aligner(0)
    result = {"card": card(), "chunk_mb": args.chunk_mb, "formats": {}}
    cores = os.cpu_count() or 1
    with tempfile.TemporaryDirectory() as tmp:
        for fmt, unit in streams.items():
            data = unit * max(1, (args.mb << 20) // len(unit))
            path = os.path.join(tmp, "out." + fmt)
            runs = []
            for _ in range(args.repeat + 1):   # the first run warms up
                t0 = time.perf_counter()
                w = a.bgzf_writer(path, chunk_bytes=args.chunk_mb << 20)
                t1 = time.perf_counter()
                for i in range(0, len(data), 8 << 20):
                    w.write(data[i:i + (8 << 20)])
                w.close()
                t2 = time.perf_counter()
                st = w.stats()
                runs.append((t2 - t0, st["device_ms"], st["bytes_out"], t2 - t1))
            runs = runs[1:]
            payload = runs[0][2] - 26 * ((len(data) + BLOCK - 1) // BLOCK)
            prefix = data[:args.zlib_mb << 20]
            pieces = [prefix[i:i + BLOCK] for i in range(0, len(prefix), BLOCK)]
            scale = len(data) / len(prefix)
            z = {}
            for level in (1, 6):
                s1, t1 = zlib_pass(pieces, level, 1)
                sn, tn = zlib_pass(pieces, level, cores)
                assert s1 == sn
                z[f"zlib{level}"] = {"payload_bytes_scaled": round(s1 * scale), "gbps_1_thread": len(prefix) / t1 / 1e9,
                                     f"gbps_{cores}_cores": len(prefix) / tn / 1e9}
            result["formats"][fmt] = {
                "input_bytes": len(data),
                "device_deflate_gbps": [len(data) / (r[1] * 1e6) for r in runs],
                "end_to_end_gbps": [len(data) / r[0] / 1e9 for r in runs],
                "after_open_gbps": [len(data) / r[3] / 1e9 for r in runs],
                "open_s": [r[0] - r[3] for r in runs],
                "payload_bytes": payload,
                "ratio_vs_zlib1": payload / z["zlib1"]["payload_bytes_scaled"],
                "ratio_vs_zlib6": payload / z["zlib6"]["payload_bytes_scaled"],
                **z,
            }
    a.close()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
