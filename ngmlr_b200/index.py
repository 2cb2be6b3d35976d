"""Pre-index a reference on the GPU for ngmlr:

    python -m ngmlr_b200.index REF.fa [-k 13] [--kmer-skip 2] [--gpu 0]

writes REF.fa-enc.2.ngm and REF.fa-ht-<k>-<skip>.2.ngm next to the FASTA file (plain or gzip), byte-compatible with
the files ngmlr writes itself, so that an unmodified ngmlr started with the same -r / -k / --kmer-skip reads them
instead of building its index on the CPU. Existing caches are kept unless --rebuild is given. Prints the phase times.
"""
import argparse
import sys

from .aligner import B200Aligner


def main(argv=None):
    ap = argparse.ArgumentParser(prog="python -m ngmlr_b200.index", description=__doc__.split("\n\n")[0])
    ap.add_argument("fasta", help="reference FASTA / FASTQ file, plain or gzip (ngmlr -r)")
    ap.add_argument("-k", "--kmer-length", type=int, default=13, help="k-mer length (ngmlr -k, default 13)")
    ap.add_argument("--kmer-skip", type=int, default=2, help="k-mers skipped between table entries (default 2)")
    ap.add_argument("--gpu", type=int, default=0, help="CUDA device (default 0)")
    ap.add_argument("--rebuild", action="store_true", help="ignore existing cache files and write new ones")
    a = ap.parse_args(argv)
    try:
        al = B200Aligner(a.gpu)
    except RuntimeError as e:
        print(f"error: {e}", file=sys.stderr)
        return 1
    try:
        ref = al.load_reference(a.fasta, k=a.kmer_length, kmer_skip=a.kmer_skip, rebuild=a.rebuild)
    except RuntimeError as e:
        print(f"error: {e}", file=sys.stderr)
        return 1
    finally:
        al.close()
    enc = f"{a.fasta}-enc.2.ngm"
    idx = f"{a.fasta}-ht-{a.kmer_length}-{a.kmer_skip}.2.ngm"
    state = lambda read, written: "read" if read else ("written" if written else "NOT written")
    print(f"{len(ref.names)} contigs, {ref.concat_len} positions")
    print(f"{enc}: {state(ref.reference_read, ref.reference_written)}")
    print(f"{idx}: {state(ref.index_read, ref.index_written)}")
    print("phases (ms): " + ", ".join(f"{k} {v:.1f}" for k, v in ref.ms.items()))
    return 0 if (ref.reference_read or ref.reference_written) and (ref.index_read or ref.index_written) else 2


if __name__ == "__main__":
    sys.exit(main())
