"""Where the IAlignment object and the resident pipeline part ways on bench.py's workload.

Builds bench.py's workload (config, seed 2, first --intervals intervals), runs the resident pipeline on all of it
(intervals_upload -> run -> fetch: the first attempt of every interval, as bench.py's `gpu_first`), then pushes the
same problems through CreateAlignment -> IAlignment::BatchAlign (ngmlr_b200_plugin_time_batch_align) and reports,
per differing interval, both sides' Score bits, ret and CIGAR+MD digest next to the oracle's single_align, how many
intervals differ and whether the plugin failed the whole batch, the plugin context's last error and batch statistics,
and device memory in use before and after the batch.

    python scripts/ialignment_check.py --config ont                 # the plugin's context alone
    python scripts/ialignment_check.py --config ont --contexts 4    # bench.py's resident contexts alive beside it

Needs a CUDA device; the oracle (oracle/liboracle.so) checks the first --oracle differing intervals."""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def fnv(s):
    c = 2166136261
    for ch in s.encode():
        c = ((c ^ ch) * 16777619) & 0xffffffff
    return c


def mem_in_use_gb(torch):
    free, total = torch.cuda.mem_get_info()
    return round((total - free) / 1e9, 3)


def plugin_batch(lib, probs, gpu_id):
    """One CreateAlignment object, one BatchAlign of every problem; -> (rets, score bits, crc, last error, stats)."""
    from ngmlr_b200 import PackedBatch, _lib
    lib.CreateAlignment.restype = C.c_void_p
    lib.CreateAlignment.argtypes = [C.c_int]
    lib.DeleteAlignment.argtypes = [C.c_void_p]
    i32p, i64p, u32p = C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.POINTER(C.c_uint32)
    lib.ngmlr_b200_plugin_time_batch_align.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_char_p),
                                                       C.POINTER(C.c_char_p), i32p, i32p, i64p, i32p, i32p, C.c_int,
                                                       C.POINTER(C.c_double), i32p, u32p, u32p]
    pb = PackedBatch.from_problems(probs)
    a = lib.CreateAlignment(gpu_id)
    assert a, "CreateAlignment failed"
    ctx = lib.ngmlr_b200_plugin_context(a)
    n = pb.n
    rets = np.zeros(n, np.int32)
    bits = np.zeros(n, np.uint32)
    crc = np.zeros(n, np.uint32)
    sec = C.c_double(0)
    args = pb.c_args()
    rc = lib.ngmlr_b200_plugin_time_batch_align(a, n, args[1], args[3], args[5], args[6], args[7], args[8], args[9], 1,
                                                C.byref(sec), rets.ctypes.data_as(i32p), bits.ctypes.data_as(u32p),
                                                crc.ctypes.data_as(u32p))
    err = lib.ngmlr_b200_last_error(ctx)
    st = _lib.BatchStats()
    lib.ngmlr_b200_convex_stats(ctx, C.byref(st))
    stats = {k: getattr(st, k) for k in ("fill_launches", "dir_bytes", "cells", "fill_ms")}
    lib.DeleteAlignment(a)
    return rc, rets, bits, crc, (err.decode() if err else ""), stats, sec.value


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="ont")
    ap.add_argument("--reads", type=int, default=8192, help="reads of bench.py's workload (its --reads)")
    ap.add_argument("--intervals", type=int, default=2048, help="leading intervals pushed through the plugin")
    ap.add_argument("--contexts", type=int, default=0,
                    help="resident contexts kept alive beside the plugin, each with its slice uploaded and run "
                         "(bench.py: 4, plus one on the whole batch)")
    ap.add_argument("--oracle", type=int, default=4, help="differing intervals also checked against the oracle")
    ap.add_argument("--gpu", type=int, default=0)
    args = ap.parse_args()

    import torch
    import bench
    from ngmlr_b200 import B200Aligner, IntervalBatch, PackedReads, _lib
    torch.cuda.set_device(args.gpu)
    cfg = bench.CONFIGS[args.config]
    bargs = argparse.Namespace(genome_mb=cfg["genome_mb"])
    genome, contig_len, enc_ref, _t = bench.build_reference(bargs, cfg, 0, 1, torch.device("cuda", args.gpu))
    wl = bench.Workload(genome, contig_len, enc_ref, args.reads, 2, cfg)
    k = min(args.intervals, len(wl.ivs))
    ivs = wl.ivs[:k]
    out = {"config": args.config, "intervals": k, "contexts": args.contexts}

    # the resident pipeline on the whole batch (bench.py's solo context: gpu_first)
    al = B200Aligner(args.gpu)
    al.set_reference(enc_ref)
    al.build_index(enc_ref)
    al.reads_upload(PackedReads(wl.reads))
    al.intervals_upload(IntervalBatch(wl.tasks(wl.ivs)))
    al.run()
    gpu_first = [r.as_dict() for r in al.fetch()[:k]]
    als = [al]
    if args.contexts:
        # bench.py's contexts: the solo context is context 0; each takes every S-th read, runs its slice resident
        # and then end to end (compute_alignments), and all of them stay alive while the plugin runs
        for _ in range(1, args.contexts):
            a_ = B200Aligner(args.gpu)
            a_.share_reference(al)
            als.append(a_)
        for j, a_ in enumerate(als):
            r_, iv_, rmap = wl.slice(j, args.contexts)
            a_.reads_upload(PackedReads(r_))
            a_.intervals_upload(IntervalBatch(wl.tasks(iv_, rmap)))
            a_.run()
            a_.compute_alignments(IntervalBatch(wl.tasks(iv_, rmap)))
    else:
        al.close()
        als = []
    torch.cuda.synchronize()

    lib = _lib.load()
    probs = [iv.problem(wl.genome, wl.reads) for iv in ivs]
    out["problems_longer_than_32767"] = sum(1 for p in probs if len(p.qry) > 32767)
    out["problems_longer_than_65535"] = sum(1 for p in probs if len(p.qry) > 65535)
    out["mem_in_use_gb_before"] = mem_in_use_gb(torch)
    rc, rets, bits, crc, err, stats, sec = plugin_batch(lib, probs, args.gpu)
    out["mem_in_use_gb_after"] = mem_in_use_gb(torch)
    out.update(plugin_rc=rc, plugin_last_error=err, plugin_stats=stats, plugin_batch_s=round(sec, 3))
    minus_one = int(np.float32(-1.0).view(np.uint32))
    out["plugin_all_score_minus_one"] = bool(np.all(bits == minus_one))
    differ = []
    for i, g in enumerate(gpu_first):
        if g["ret"] < 0:
            if rets[i] >= 0:
                differ.append(i)
            continue
        if int(bits[i]) != g["score_bits"] or int(crc[i]) != fnv(g["cigar"] + g["md"]):
            differ.append(i)
    out["differing"] = len(differ)
    out["first_differing"] = differ[:16]
    rows = []
    if differ:
        from oracle_lib import Oracle
        orc = Oracle()
        for i in differ[:args.oracle]:
            p = probs[i]
            g = gpu_first[i]
            w = orc.single_align(p.ref, p.qry, p.offsets, p.lengths, p.ext_qstart, p.ext_qend)
            rows.append({"interval": i, "read_len": len(p.qry), "ref_len": len(p.ref),
                         "cells": int(np.maximum(np.asarray(p.lengths), 0).sum()),
                         "plugin": {"ret": int(rets[i]), "score_bits": int(bits[i]), "cigar_md_fnv": int(crc[i])},
                         "resident": {"ret": g["ret"], "score_bits": g["score_bits"],
                                      "cigar_md_fnv": fnv(g["cigar"] + g["md"]), "cigar": g["cigar"][:60],
                                      "md": g["md"][:60]},
                         "oracle": {"ret": w["ret"], "score_bits": w["score_bits"],
                                    "cigar_md_fnv": fnv(w["cigar"] + w["md"]) if w["ret"] >= 0 else None,
                                    "cigar": w["cigar"][:60], "md": w["md"][:60]}})
    out["rows"] = rows
    print(json.dumps(out, indent=1))
    for a_ in als:
        a_.close()


if __name__ == "__main__":
    main()
