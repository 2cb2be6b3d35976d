// ngmlr_b200/csrc/reference_load.cu -- ngmlr's start-up as one call (ngmlr_b200_load_reference): the reference and
// its k-mer index from ngmlr's cache files, or from the FASTA file with the encoding and the index built on the device,
// in the order of _SequenceProvider::Init (src/SequenceProvider.cpp:246-424) and the CompactPrefixTable constructor
// (src/PrefixTable.cpp:97-128). Host glue around entry points that exist on their own: fasta.cpp reads the file,
// cs_encode_reference / cs_build_index run on the device, ngm_files.cpp reads and writes the caches.
#include <sys/stat.h>
#include <unistd.h>

#include "fasta.h"
#include "runtime.h"

using namespace nb;

namespace {

bool file_exists(const std::string& p) {
  struct stat st;
  return stat(p.c_str(), &st) == 0;
}

// Writes a cache under a temporary name and renames it: an interrupted write never leaves a truncated cache that a
// later start would read (ngmlr trusts the encoded reference's header).
template <typename W>
bool write_cache(const std::string& path, W write) {
  const std::string tmp = path + ".tmp" + std::to_string((long)getpid());
  if (write(tmp.c_str()) != 0) {
    unlink(tmp.c_str());
    return false;
  }
  if (rename(tmp.c_str(), path.c_str()) != 0) {
    unlink(tmp.c_str());
    return false;
  }
  return true;
}

// No reference and no index on the context (a load that failed after it reached the device).
void drop_reference(CsState* cs) {
  cs->enc_bytes = 0;
  cs->concat_len = 0;
  cs->ref_starts.clear();
  cs->index_len = 0;
  cs->n_pos = 0;
  cs->rn = 0;
  cs->reads_searched = false;
  cs->contig_names.clear();
}

}  // namespace

extern "C" {

int ngmlr_b200_load_reference(ngmlr_b200_ctx* ctx, const char* fasta_path, const ngmlr_b200_reference_options* opts,
                              int32_t* n_contigs, uint64_t* concat_len, int32_t* flags) {
  if (!ctx) return -1;
  const double t0 = now_ms();
  ngmlr_b200_reference_options o = {13, 2, 4, 1000, 0, 0};
  if (opts) o = *opts;
  if (!fasta_path) return ctx->fail("load_reference: no FASTA path");
  if (o.k < 1 || o.k > 15 || o.kmer_skip < 0 || o.bin_shift < 0 || o.bin_shift > 31 || o.max_prefix_freq < 1)
    return ctx->fail("load_reference: bad options (k in 1..15, kmer_skip >= 0, bin_shift in 0..31, max_prefix_freq >= 1)");
  if (!file_exists(fasta_path)) return ctx->fail("load_reference: cannot open %s", fasta_path);
  const std::string enc_path = std::string(fasta_path) + "-enc.2.ngm";
  const std::string idx_path =
      std::string(fasta_path) + "-ht-" + std::to_string(o.k) + "-" + std::to_string(o.kmer_skip) + ".2.ngm";
  int32_t fl = 0;
  // ---- 1. the reference on the host: nothing on the context changes before it passed every check ----
  FastaText fa;
  PinBuf<uint8_t> enc_host;
  std::vector<std::string> names;
  std::vector<uint64_t> starts, lens;
  uint64_t used = 0, cl = 0;
  const bool ref_cached = !o.rebuild && file_exists(enc_path);
  if (ref_cached) {
    uint32_t n = 0;
    uint64_t alloc = 0;
    if (ngmlr_b200_ngm_read_reference(enc_path.c_str(), &n, &used, &alloc, nullptr, nullptr, nullptr, nullptr) != 0 ||
        n == 0 || used == 0)
      return ctx->fail("load_reference: %s is not a valid encoded reference; delete it or load with rebuild",
                       enc_path.c_str());
    cl = 2 * used - 1;
    if (!index_build_fits(cl, (int)std::min<uint32_t>(n, 1u << 30), o.kmer_skip))
      return ctx->fail("load_reference: %s holds %llu positions; one k-mer table unit holds at most %llu (and at most "
                       "2^31 k-mer callbacks)", enc_path.c_str(), (unsigned long long)cl, INDEX_MAX_CONCAT_LEN);
    std::vector<char> nm((size_t)n * 101);
    std::vector<uint32_t> len32(n);
    starts.resize(n);
    if (enc_host.reserve(used) != cudaSuccess) return ctx->fail("load_reference: cannot allocate %llu bytes of host memory", (unsigned long long)used);
    if (ngmlr_b200_ngm_read_reference(enc_path.c_str(), &n, &used, &alloc, starts.data(), len32.data(), nm.data(),
                                      enc_host.p) != 0)
      return ctx->fail("load_reference: %s is truncated; delete it or load with rebuild", enc_path.c_str());
    for (uint32_t i = 0; i < n; ++i) {
      lens.push_back(len32[i]);
      names.emplace_back(nm.data() + (size_t)i * 101);
      if ((i && starts[i] < starts[i - 1] + lens[i - 1]) || starts[i] + lens[i] > cl)
        return ctx->fail("load_reference: %s has an inconsistent contig table", enc_path.c_str());
    }
    fl |= NGMLR_B200_LOAD_REFERENCE_READ;
  } else {
    std::string err;
    if (read_fasta(fasta_path, true, INDEX_MAX_CONCAT_LEN, fa, err) != 0) return ctx->fail("load_reference: %s", err.c_str());
    std::vector<uint64_t> all;
    for (const FastaRecord& r : fa.recs) {
      all.push_back(r.len);
      if (r.len > 10) names.push_back(r.name.substr(0, 100));  // RefIdx::name (src/SequenceProvider.cpp:353-355)
    }
    if (names.empty()) return ctx->fail("load_reference: %s holds no sequence of more than 10 bases", fasta_path);
    cl = concat_len_of(all);
    if (!index_build_fits(cl, (int)names.size(), o.kmer_skip))
      return ctx->fail("load_reference: %llu positions give more than 2^31 k-mer callbacks at kmer_skip %d",
                       (unsigned long long)cl, o.kmer_skip);
  }
  const double t1 = now_ms();
  // ---- 2. install: from here on a failure leaves the context without reference and index ----
  CsState* cs = cs_state(ctx, true);
  // a context that used another one's arrays (cs_share_reference) gets its own instead of overwriting them
  for (DevBuf<uint8_t>* b : {&cs->d_enc}) if (b->borrowed) b->release();
  for (DevBuf<uint32_t>* b : {&cs->d_tab, &cs->d_used, &cs->d_pos}) if (b->borrowed) b->release();
  if (cs->d_rci.borrowed) cs->d_rci.release();
  if (cs->d_ref_starts.borrowed) cs->d_ref_starts.release();
  auto undo = [&]() {
    drop_reference(cs);
    return -1;
  };
  int rc;
  if (ref_cached) {
    std::vector<uint64_t> rs(starts);
    rs.push_back(starts.back() + lens.back() + 1000);  // refStartPos' artificial last entry
    rc = ngmlr_b200_cs_set_reference(ctx, enc_host.p, used, cl);
    if (rc == 0) rc = ngmlr_b200_set_ref_starts(ctx, rs.data(), (int)rs.size());
    if (rc != 0) return undo();
  } else {
    const size_t n = fa.recs.size();
    std::vector<const char*> seqs(n);
    std::vector<uint64_t> all(n);
    for (size_t i = 0; i < n; ++i) {
      seqs[i] = fa.text + fa.recs[i].offset;
      all[i] = fa.recs[i].len;
    }
    starts.resize(n);
    lens.resize(n);
    int32_t kept = 0;
    uint64_t nbytes = 0, cl2 = 0;
    rc = ngmlr_b200_cs_encode_reference(ctx, (int)n, seqs.data(), all.data(), &kept, starts.data(), lens.data(),
                                        &nbytes, &cl2);
    if (rc != 0) return undo();
    starts.resize(kept);
    lens.resize(kept);
    used = nbytes;
    fa.release_text();
  }
  const double t2 = now_ms();
  if (!ref_cached && !o.skip_write) {
    if (enc_host.reserve(used) != cudaSuccess) return (ctx->fail("load_reference: out of pinned host memory"), undo());
    if (ngmlr_b200_cs_get_reference(ctx, enc_host.p, used, nullptr, nullptr) != 0) return undo();
    std::vector<uint32_t> len32(lens.begin(), lens.end());
    std::vector<const char*> nm;
    for (const std::string& s : names) nm.push_back(s.c_str());
    const uint64_t alloc = fa.alloc_bytes();
    if (write_cache(enc_path, [&](const char* p) {
          return ngmlr_b200_ngm_write_reference(p, enc_host.p, used, alloc, (int)starts.size(), starts.data(),
                                                len32.data(), nm.data());
        }))
      fl |= NGMLR_B200_LOAD_REFERENCE_WRITTEN;
  }
  enc_host.release();
  const double t3 = now_ms();
  // ---- 3. the k-mer index ----
  bool idx_cached = false;
  if (!o.rebuild && file_exists(idx_path)) {
    int32_t k2 = 0, s2 = 0;
    uint32_t il = 0, np = 0;
    uint64_t off = 0;
    if (ngmlr_b200_ngm_read_index(idx_path.c_str(), &k2, &s2, &il, &np, &off, nullptr, nullptr) == 0 && k2 == o.k &&
        s2 == o.kmer_skip && il == (1u << (2 * o.k)) + 1u && off == 0) {
      PinBuf<uint8_t> packed;
      PinBuf<uint32_t> pos;
      if (packed.reserve((size_t)il * 5) != cudaSuccess || pos.reserve((size_t)np + 1) != cudaSuccess)
        return (ctx->fail("load_reference: out of pinned host memory"), undo());
      if (ngmlr_b200_ngm_read_index(idx_path.c_str(), &k2, &s2, &il, &np, &off, packed.p, pos.p) == 0) {
        if (ngmlr_b200_cs_set_index(ctx, packed.p, il, pos.p, np, 0, o.k, o.bin_shift) != 0) return undo();
        idx_cached = true;
        fl |= NGMLR_B200_LOAD_INDEX_READ;
      }
    }
  }
  const double t4a = now_ms();
  double t5 = t4a;
  if (!idx_cached) {
    uint32_t np = 0;
    if (ngmlr_b200_cs_build_index(ctx, starts.data(), lens.data(), (int)starts.size(), o.k, o.kmer_skip, o.bin_shift,
                                  o.max_prefix_freq, &np) != 0)
      return undo();
    t5 = now_ms();
    if (!o.skip_write) {
      uint32_t il = 0;
      PinBuf<uint8_t> packed;
      PinBuf<uint32_t> pos;
      if (ngmlr_b200_cs_get_index(ctx, &il, &np, nullptr, nullptr) != 0) return undo();
      if (packed.reserve((size_t)il * 5) != cudaSuccess || pos.reserve((size_t)np + 1) != cudaSuccess)
        return (ctx->fail("load_reference: out of pinned host memory"), undo());
      if (ngmlr_b200_cs_get_index(ctx, nullptr, nullptr, packed.p, pos.p) != 0) return undo();
      if (write_cache(idx_path, [&](const char* p) {
            return ngmlr_b200_ngm_write_index(p, o.k, o.kmer_skip, packed.p, il, pos.p, np, 0);
          }))
        fl |= NGMLR_B200_LOAD_INDEX_WRITTEN;
    }
  }
  const double t6 = now_ms();
  cs->rn = 0;  // resident candidates belonged to the previous reference
  cs->reads_searched = false;
  cs->contig_names = names;
  cs->contig_start = starts;
  cs->contig_len = lens;
  cs->contig_name_ptrs.clear();
  for (const std::string& s : cs->contig_names) cs->contig_name_ptrs.push_back(s.c_str());
  const float ms[6] = {(float)(t1 - t0), (float)(t2 - t1), (float)(t3 - t2), (float)((idx_cached ? t4a : t5) - t3),
                       (float)(t6 - (idx_cached ? t4a : t5)), (float)(t6 - t0)};
  memcpy(cs->load_ms, ms, sizeof ms);
  if (n_contigs) *n_contigs = (int32_t)starts.size();
  if (concat_len) *concat_len = cs->concat_len;
  if (flags) *flags = fl;
  return 0;
}

int ngmlr_b200_reference_contigs(ngmlr_b200_ctx* ctx, const char** names, int32_t* name_lens, uint64_t* starts,
                                 uint64_t* lens) {
  if (!ctx) return -1;
  CsState* cs = cs_state(ctx, false);
  if (!cs || !cs->enc_bytes || cs->contig_names.empty())
    return ctx->fail("reference_contigs: the context's reference was not loaded with load_reference");
  const size_t n = cs->contig_names.size();
  for (size_t i = 0; i < n; ++i) {
    if (names) names[i] = cs->contig_name_ptrs[i];
    if (name_lens) name_lens[i] = (int32_t)cs->contig_names[i].size();
    if (starts) starts[i] = cs->contig_start[i];
    if (lens) lens[i] = cs->contig_len[i];
  }
  return (int)n;
}

// Milliseconds of the phases of the context's last load_reference: read (cache file or FASTA parse), install (H2D +
// device encoding, or H2D of the cached genome), reference cache write (D2H + file), index (device build, or cache
// read + H2D), index cache write (D2H + file), total.
int ngmlr_b200_load_reference_ms(ngmlr_b200_ctx* ctx, float* ms) {
  if (!ctx || !ms) return -1;
  CsState* cs = cs_state(ctx, false);
  if (!cs) return ctx->fail("load_reference_ms: no load");
  memcpy(ms, cs->load_ms, sizeof cs->load_ms);
  return 0;
}

// Test hook, no context: the records read_fasta yields (host memory, not page-locked). Counts always; names (their
// name_lens concatenated), record lengths and the concatenated sequence text where the pointers are not NULL.
// Returns 0, or < 0 with the message in err.
int ngmlr_b200_debug_read_fasta(const char* path, uint64_t max_concat_len, int64_t* n_recs, uint64_t* text_size,
                                uint64_t* names_size, uint64_t* alloc_bytes, int64_t* name_lens, uint64_t* rec_lens,
                                char* names, char* text, char* err, int err_cap) {
  FastaText fa;
  std::string e;
  const int rc = read_fasta(path, false, max_concat_len, fa, e);
  if (rc != 0) {
    if (err && err_cap > 0) snprintf(err, (size_t)err_cap, "%s", e.c_str());
    return rc;
  }
  uint64_t nsz = 0;
  for (size_t i = 0; i < fa.recs.size(); ++i) {
    const FastaRecord& r = fa.recs[i];
    if (name_lens) name_lens[i] = (int64_t)r.name.size();
    if (rec_lens) rec_lens[i] = r.len;
    if (names) memcpy(names + nsz, r.name.data(), r.name.size());
    nsz += r.name.size();
  }
  if (text && fa.size) memcpy(text, fa.text, fa.size);
  if (n_recs) *n_recs = (int64_t)fa.recs.size();
  if (text_size) *text_size = fa.size;
  if (names_size) *names_size = nsz;
  if (alloc_bytes) *alloc_bytes = fa.alloc_bytes();
  return 0;
}

}  // extern "C"
