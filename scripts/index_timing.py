"""Time ngmlr's start-up through ngmlr_b200_load_reference on a seeded synthetic genome (default 3 Gb in 24 contigs):
FASTA parse, H2D + device encoding, encoded-reference write, device k-mer index build and index write, with the
card's name and power limit read in the same run and the peak device memory in use during the load. For the CPU side
it runs the reference's own build (ref_cs_init_save of oracle/_ref/libngmlr_full.so) and the device load on a smaller
genome (--cpu-mbp) that the CPU build finishes in reasonable time.

    python scripts/index_timing.py [--gbp 3] [--contigs 24] [--cpu-mbp 50] [--out DIR]

Phase times are host clocks around work that ends in a device synchronise (ngmlr_b200_load_reference_ms); the device
index build alone is also timed with CUDA events (ngmlr_b200_cs_last_build_ms)."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
FULL = os.path.join(ROOT, "oracle", "_ref", "libngmlr_full.so")


def write_genome(path, total, n_contigs, seed):
    """Random ACGT contigs (one N run each), 60 bases per line."""
    rng = np.random.default_rng(seed)
    sizes = np.full(n_contigs, total // n_contigs, dtype=np.int64)
    sizes[: total % n_contigs] += 1
    lut = np.frombuffer(b"ACGT", dtype=np.uint8)
    with open(path, "wb") as f:
        for i, n in enumerate(sizes):
            f.write(f">chr{i + 1} synthetic contig {i + 1}\n".encode())
            left = int(n)
            while left:
                m = min(left, 60 * 2_000_000)
                s = lut[rng.integers(0, 4, m, dtype=np.uint8)]
                if left == n:
                    s[m // 3: m // 3 + 10_000] = ord("N")
                full = m // 60
                body = np.empty((full, 61), dtype=np.uint8)
                body[:, :60] = s[: full * 60].reshape(full, 60)
                body[:, 60] = ord("\n")
                f.write(body.tobytes())
                if m % 60:
                    f.write(s[full * 60:].tobytes() + b"\n")
                left -= m
    return int(sizes.sum())


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def load(path, gpu):
    """One load_reference on a fresh context, with the peak device memory in use (all processes) sampled every 2 ms."""
    import torch
    from ngmlr_b200 import B200Aligner
    torch.cuda.init()
    free0, total = torch.cuda.mem_get_info(gpu)
    peak = [0]
    done = threading.Event()

    def sample():
        while not done.is_set():
            peak[0] = max(peak[0], total - torch.cuda.mem_get_info(gpu)[0])
            time.sleep(0.002)

    th = threading.Thread(target=sample)
    th.start()
    t0 = time.perf_counter()
    a = B200Aligner(gpu)
    try:
        ref = a.load_reference(path)
        wall = (time.perf_counter() - t0) * 1e3
        build_ms = float(a.lib.ngmlr_b200_cs_last_build_ms(a.h))
    finally:
        a.close()
        done.set()
        th.join()
    return {"contigs": len(ref.names), "positions": ref.concat_len, "phases_ms": ref.ms, "wall_ms_with_context": wall,
            "index_build_kernel_ms_cuda_events": build_ms,
            "files": {"reference_written": ref.reference_written, "index_written": ref.index_written},
            "device_mem_in_use_before_GB": (total - free0) / 1e9, "device_mem_in_use_peak_GB": peak[0] / 1e9,
            "device_mem_total_GB": total / 1e9, "memory_sample_interval_ms": 2}


def reference_cpu_build(path):
    code = "import ctypes, sys; lib = ctypes.CDLL(sys.argv[1]); sys.exit(lib.ref_cs_init_save(sys.argv[2].encode()))"
    t0 = time.perf_counter()
    r = subprocess.run([sys.executable, "-c", code, FULL, path], capture_output=True, text=True)
    return {"ms": (time.perf_counter() - t0) * 1e3, "returncode": r.returncode}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--gbp", type=float, default=3.0)
    ap.add_argument("--contigs", type=int, default=24)
    ap.add_argument("--cpu-mbp", type=float, default=50.0)
    ap.add_argument("--gpu", type=int, default=0)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    a = ap.parse_args()
    out = {"gpu": gpu_info()}
    work = tempfile.mkdtemp(prefix="index_timing_")
    try:
        big = os.path.join(work, "genome.fa")
        t0 = time.perf_counter()
        out["genome_bases"] = write_genome(big, int(a.gbp * 1e9), a.contigs, a.seed)
        out["genome_write_s"] = time.perf_counter() - t0
        out["fasta_bytes"] = os.path.getsize(big)
        out["device_load"] = load(big, a.gpu)
        for f in os.listdir(work):
            os.remove(os.path.join(work, f))
        small = os.path.join(work, "small.fa")
        out["small_genome_bases"] = write_genome(small, int(a.cpu_mbp * 1e6), 4, a.seed + 1)
        out["small_device_load"] = load(small, a.gpu)
        for f in os.listdir(work):
            if f != "small.fa":
                os.remove(os.path.join(work, f))
        out["small_reference_cpu_build"] = reference_cpu_build(small) if os.path.exists(FULL) else "not measured"
    finally:
        shutil.rmtree(work, ignore_errors=True)
    text = json.dumps(out, indent=1)
    print(text)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "index_timing.json"), "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
