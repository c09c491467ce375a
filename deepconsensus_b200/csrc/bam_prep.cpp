// Feature construction from BAM, htslib-free (and the producer half of the packed rows): the part of
// `deepconsensus run` that sits in front of the model path, as host C++ behind the C ABI (include/dcb200.h "dcb_prep_*",
// "dcb_bamw_*").
//
//   BGZF / BAM reader            what pysam.AlignmentFile does for pre_lib.py:50-91,1279-1367 (SAM/BAM spec v1.6 section 4)
//   SubreadGrouper               pre_lib.py:50-91     mapped subreads of one ZMW (`zm` tag), in file order
//   trim_insertions              pre_lib.py:1061-1125 insertions longer than ins_trim removed from seq / cigar / pw / ip
//   expand_clip_indent           pre_lib.py:1128-1239 gaps at deletions, soft clips removed, indent to the CCS start,
//                                                     pw / ip reversed for reverse-strand alignments
//   construct_ccs_read           pre_lib.py:966-998
//   space_out_subreads           pre_lib.py:1242-1276 columns opened in every read wherever any read has an insertion
//   DcExample.iter_examples /    pre_lib.py:625-744   windows of max_length columns, padding, the [R, L] feature rows --
//   extract_features                                  written as float32 rows AND as packed rows (dcb_pack_rows' format)
//   unaligned BAM writer         quick_inference.py:740-760,892-897  (ec, np, rq, RG, zm tags; the CCS BAM's header)
//
// Pinned against the reference's own fixture: the windows built here from testdata/human_1m/{subreads_to_ccs,ccs}.bam
// equal, value for value, the 1 593 examples of testdata/human_1m/tf_examples/inference/inference.tfrecord.gz that the
// reference's preprocess wrote from the same BAMs (tests/test_bam_prep.py).
#include <ctype.h>
#include <math.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <zlib.h>

#include <algorithm>
#include <condition_variable>
#include <deque>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../../include/dcb200.h"
#include "common.h"

namespace {

thread_local std::string g_prep_error;

int pfail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  g_prep_error = buf;
  return code;
}

// ----------------------------------------------------------------------------------------------- BGZF reader
struct Bgzf {
  FILE* f = nullptr;
  std::vector<uint8_t> block;   // inflated current block
  size_t pos = 0;
  bool fail = false;
  ~Bgzf() { if (f) fclose(f); }
  bool next_block() {
    uint8_t h[12];
    size_t n = fread(h, 1, 12, f);
    if (n == 0) return false;                       // clean EOF
    if (n != 12 || h[0] != 31 || h[1] != 139 || h[2] != 8 || !(h[3] & 4)) { fail = true; return false; }
    const int xlen = h[10] | (h[11] << 8);
    std::vector<uint8_t> extra(xlen);
    if (fread(extra.data(), 1, xlen, f) != (size_t)xlen) { fail = true; return false; }
    int bsize = -1;
    for (int i = 0; i + 4 <= xlen;) {
      const int slen = extra[i + 2] | (extra[i + 3] << 8);
      if (extra[i] == 'B' && extra[i + 1] == 'C' && slen == 2) bsize = extra[i + 4] | (extra[i + 5] << 8);
      i += 4 + slen;
    }
    if (bsize < 0) { fail = true; return false; }
    const int clen = bsize - xlen - 19;
    if (clen < 0) { fail = true; return false; }
    std::vector<uint8_t> comp(clen + 8);
    if (fread(comp.data(), 1, clen + 8, f) != (size_t)clen + 8) { fail = true; return false; }
    const uint32_t isize = comp[clen + 4] | (comp[clen + 5] << 8) | (comp[clen + 6] << 16) | ((uint32_t)comp[clen + 7] << 24);
    block.resize(isize);
    pos = 0;
    if (isize == 0) return true;                    // the EOF marker block (or an empty block)
    z_stream zs;
    memset(&zs, 0, sizeof zs);
    if (inflateInit2(&zs, -15) != Z_OK) { fail = true; return false; }
    zs.next_in = comp.data(); zs.avail_in = clen;
    zs.next_out = block.data(); zs.avail_out = isize;
    const int rc = inflate(&zs, Z_FINISH);
    inflateEnd(&zs);
    if (rc != Z_STREAM_END || zs.total_out != isize) { fail = true; return false; }
    const uint32_t crc = comp[clen] | (comp[clen + 1] << 8) | (comp[clen + 2] << 16) | ((uint32_t)comp[clen + 3] << 24);
    if ((uint32_t)crc32(0, block.data(), isize) != crc) { fail = true; return false; }
    return true;
  }
  // 1 = ok, 0 = clean EOF before any byte, -1 = error / truncated
  int read(void* dst, size_t n) {
    uint8_t* d = static_cast<uint8_t*>(dst);
    size_t got = 0;
    while (got < n) {
      if (pos == block.size()) {
        if (!next_block()) return (got == 0 && !fail) ? 0 : -1;
        continue;
      }
      const size_t take = std::min(n - got, block.size() - pos);
      memcpy(d + got, block.data() + pos, take);
      pos += take; got += take;
    }
    return 1;
  }
  // Positions the reader at a BGZF virtual offset: the compressed block starts at voff >> 16, the record at byte
  // voff & 0xffff of its inflated contents.
  bool seek(uint64_t voff) {
    fail = false;
    if (fseeko(f, (off_t)(voff >> 16), SEEK_SET) != 0 || !next_block()) { fail = true; return false; }
    pos = voff & 0xffff;
    if (pos > block.size()) { fail = true; return false; }
    return true;
  }
};

struct Tag { char type = 0, sub = 0; const uint8_t* p = nullptr; size_t count = 0; };

struct BamRecord {
  std::string qname, seq;
  int32_t refid = -1, pos = -1;
  uint16_t flag = 0;
  std::vector<uint32_t> cigar;        // len << 4 | op
  std::vector<uint8_t> qual, aux;
  bool find(const char* name, Tag* t) const {
    size_t i = 0;
    const size_t n = aux.size();
    while (i + 3 <= n) {
      const bool hit = aux[i] == (uint8_t)name[0] && aux[i + 1] == (uint8_t)name[1];
      const char ty = (char)aux[i + 2];
      i += 3;
      size_t len = 0, cnt = 1;
      char sub = 0;
      switch (ty) {
        case 'A': case 'c': case 'C': len = 1; break;
        case 's': case 'S': len = 2; break;
        case 'i': case 'I': case 'f': len = 4; break;
        case 'Z': case 'H': { size_t j = i; while (j < n && aux[j]) ++j; len = j - i + 1; break; }
        case 'B': {
          if (i + 5 > n) return false;
          sub = (char)aux[i];
          cnt = aux[i + 1] | (aux[i + 2] << 8) | (aux[i + 3] << 16) | ((size_t)aux[i + 4] << 24);
          const size_t es = (sub == 'c' || sub == 'C') ? 1 : (sub == 's' || sub == 'S') ? 2 : 4;
          i += 5; len = es * cnt; break;
        }
        default: return false;
      }
      if (i + len > n) return false;
      if (hit) { t->type = ty; t->sub = sub; t->p = aux.data() + i; t->count = cnt; return true; }
      i += len;
    }
    return false;
  }
  static double scalar(const Tag& t) {
    switch (t.type) {
      case 'c': return (int8_t)t.p[0];
      case 'C': return t.p[0];
      case 's': { int16_t v; memcpy(&v, t.p, 2); return v; }
      case 'S': { uint16_t v; memcpy(&v, t.p, 2); return v; }
      case 'i': { int32_t v; memcpy(&v, t.p, 4); return v; }
      case 'I': { uint32_t v; memcpy(&v, t.p, 4); return v; }
      case 'f': { float v; memcpy(&v, t.p, 4); return v; }
      default: return 0;
    }
  }
  static double element(const Tag& t, size_t i) {
    switch (t.sub) {
      case 'c': return (int8_t)t.p[i];
      case 'C': return t.p[i];
      case 's': { int16_t v; memcpy(&v, t.p + 2 * i, 2); return v; }
      case 'S': { uint16_t v; memcpy(&v, t.p + 2 * i, 2); return v; }
      case 'i': { int32_t v; memcpy(&v, t.p + 4 * i, 4); return v; }
      case 'I': { uint32_t v; memcpy(&v, t.p + 4 * i, 4); return v; }
      case 'f': { float v; memcpy(&v, t.p + 4 * i, 4); return v; }
      default: return 0;
    }
  }
};

struct BamReader {
  Bgzf z;
  std::string header_text;
  std::vector<std::string> refs;
  std::vector<int32_t> ref_len;
  int open(const char* path) {
    z.f = fopen(path, "rb");
    if (!z.f) return pfail(DCB_ERR_INVALID, "cannot open %s", path);
    char magic[4];
    int32_t l_text, n_ref;
    if (z.read(magic, 4) != 1 || memcmp(magic, "BAM\1", 4) || z.read(&l_text, 4) != 1 || l_text < 0)
      return pfail(DCB_ERR_INVALID, "%s: not a BAM file", path);
    header_text.resize(l_text);
    if (l_text && z.read(&header_text[0], l_text) != 1) return pfail(DCB_ERR_INVALID, "%s: truncated header", path);
    while (!header_text.empty() && header_text.back() == '\0') header_text.pop_back();
    if (z.read(&n_ref, 4) != 1 || n_ref < 0) return pfail(DCB_ERR_INVALID, "%s: truncated header", path);
    for (int i = 0; i < n_ref; ++i) {
      int32_t l_name, l_ref;
      if (z.read(&l_name, 4) != 1 || l_name <= 0) return pfail(DCB_ERR_INVALID, "%s: bad reference list", path);
      std::string nm(l_name, '\0');
      if (z.read(&nm[0], l_name) != 1 || z.read(&l_ref, 4) != 1) return pfail(DCB_ERR_INVALID, "%s: bad reference list", path);
      nm.resize(strlen(nm.c_str()));
      refs.push_back(nm);
      ref_len.push_back(l_ref);
    }
    return DCB_OK;
  }
  // Appends the next record's bytes (those after its block_size) to *b, after the size checks every record gets:
  // 1 = record, 0 = EOF, < 0 = error
  int next_raw(std::vector<uint8_t>* b) {
    int32_t bs;
    const int rc = z.read(&bs, 4);
    if (rc == 0) return 0;
    if (rc < 0 || bs < 32) return pfail(DCB_ERR_INVALID, "truncated BAM record");
    if (bs > (64 << 20)) return pfail(DCB_ERR_INVALID, "implausible BAM record size %d", bs);
    const size_t at = b->size();
    b->resize(at + bs);
    if (z.read(b->data() + at, bs) != 1) return pfail(DCB_ERR_INVALID, "truncated BAM record");
    int32_t l_seq;
    uint16_t n_cig;
    memcpy(&n_cig, b->data() + at + 12, 2);
    memcpy(&l_seq, b->data() + at + 16, 4);
    if (l_seq < 0 || 32ull + (*b)[at + 8] + 4ull * n_cig + (l_seq + 1) / 2 + l_seq > (size_t)bs)
      return pfail(DCB_ERR_INVALID, "corrupt BAM record");
    return 1;
  }
  // 1 = record, 0 = EOF, < 0 = error
  int next(BamRecord* r) {
    std::vector<uint8_t> b;
    const int rc = next_raw(&b);
    if (rc <= 0) return rc;
    const int32_t bs = (int32_t)b.size();
    int32_t l_seq;
    uint16_t n_cig;
    memcpy(&r->refid, &b[0], 4);
    memcpy(&r->pos, &b[4], 4);
    const int l_name = b[8];
    memcpy(&n_cig, &b[12], 2);
    memcpy(&r->flag, &b[14], 2);
    memcpy(&l_seq, &b[16], 4);
    size_t o = 32;
    r->qname.assign(reinterpret_cast<const char*>(&b[o]), l_name ? l_name - 1 : 0);
    o += l_name;
    r->cigar.resize(n_cig);
    if (n_cig) memcpy(r->cigar.data(), &b[o], 4ull * n_cig);
    o += 4ull * n_cig;
    static const char kNt[] = "=ACMGRSVTWYHKDBN";
    r->seq.resize(l_seq);
    for (int i = 0; i < l_seq; ++i) r->seq[i] = kNt[(b[o + i / 2] >> (i & 1 ? 0 : 4)) & 15];
    o += (l_seq + 1) / 2;
    r->qual.assign(b.begin() + o, b.begin() + o + l_seq);
    o += l_seq;
    r->aux.assign(b.begin() + o, b.begin() + bs);
    return 1;
  }
};

// ----------------------------------------------------------------------------------------------- Read (pre_lib.py:111-421)
constexpr uint8_t kCMatch = 0, kCIns = 1, kCDel = 2, kCRefSkip = 3, kCSoft = 4, kCHard = 5, kCPad = 6, kCEq = 7, kCDiff = 8;
constexpr char kGap = ' ';

struct Read {
  std::string name;
  std::vector<char> bases;
  std::vector<uint8_t> cigar, pw, ip;
  float sn[4] = {0, 0, 0, 0};
  int strand = 0;                       // dc_constants.Strand: 0 unknown, 1 forward, 2 reverse
  std::vector<int32_t> ccs_idx;
  std::vector<int32_t> bq;              // base_quality_scores (CCS read only)
  bool bq_any = false;                  // `base_quality_scores.any()`: spacing only applies then (pre_lib.py:247-250)
  // spacing state (pre_lib.py:176-216)
  std::vector<int32_t> seq_indices;
  size_t idx_seq = 0;
  int32_t idx_spaced = 0;
  bool done = false;
};

// pysam get_aligned_pairs(): (query index | -1, reference index | -1) per alignment column; H and P give no column
void aligned_pairs(const std::vector<uint32_t>& cigar, int32_t pos, std::vector<int32_t>* qidx, std::vector<int32_t>* ridx) {
  int32_t q = 0, r = pos;
  for (uint32_t c : cigar) {
    const int op = c & 15;
    const int len = (int)(c >> 4);
    switch (op) {
      case kCMatch: case kCEq: case kCDiff: for (int i = 0; i < len; ++i) { qidx->push_back(q++); ridx->push_back(r++); } break;
      case kCIns: case kCSoft: for (int i = 0; i < len; ++i) { qidx->push_back(q++); ridx->push_back(-1); } break;
      case kCDel: case kCRefSkip: for (int i = 0; i < len; ++i) { qidx->push_back(-1); ridx->push_back(r++); } break;
      default: break;
    }
  }
}

// trim_insertions (pre_lib.py:1061-1125), literally: an insertion longer than ins_trim disappears from the sequence, the
// cigar and the kinetics; every other operation except a deletion advances the sequence position by its length
void trim_insertions(BamRecord* r, std::vector<double>* pw, std::vector<double>* ip, int ins_trim) {
  if (ins_trim <= 0) return;
  std::vector<uint32_t> cig;
  std::string seq;
  std::vector<char> mask(r->seq.size(), 1);
  size_t sp = 0;
  for (uint32_t c : r->cigar) {
    const int op = c & 15;
    const size_t len = c >> 4;
    if (op == kCIns && (int)len > ins_trim) {
      for (size_t i = sp; i < sp + len && i < mask.size(); ++i) mask[i] = 0;
      sp += len;
    } else {
      cig.push_back(c);
      if (op != kCDel) {
        seq += r->seq.substr(std::min(sp, r->seq.size()), len);
        sp += len;
      }
    }
  }
  const bool rev = r->flag & 16;
  auto filter = [&](std::vector<double>* v) {
    if (v->empty()) return;
    std::vector<double> out;
    const size_t n = mask.size();
    for (size_t i = 0; i < v->size() && i < n; ++i)
      if (rev ? mask[n - 1 - i] : mask[i]) out.push_back((*v)[i]);
    v->swap(out);
  };
  filter(pw);
  filter(ip);
  r->seq = seq;
  r->cigar = cig;
}

// pw / ip tags of a subread as the reference reads them (pre_lib.py:1141-1146)
void load_kinetics(const BamRecord& rec, std::vector<double>* pw, std::vector<double>* ip) {
  Tag t;
  if (rec.find("pw", &t) && t.type == 'B') { pw->resize(t.count); for (size_t i = 0; i < t.count; ++i) (*pw)[i] = BamRecord::element(t, i); }
  if (rec.find("ip", &t) && t.type == 'B') { ip->resize(t.count); for (size_t i = 0; i < t.count; ++i) (*ip)[i] = BamRecord::element(t, i); }
}

// uint8 arrays (pre_lib.py:1166-1167)
inline uint8_t kinetic_u8(double v) { return (uint8_t)v; }

inline bool op_has_column(int op) { return op == kCMatch || op == kCEq || op == kCDiff || op == kCIns || op == kCSoft || op == kCDel || op == kCRefSkip; }
inline bool op_has_query(int op) { return op == kCMatch || op == kCEq || op == kCDiff || op == kCIns || op == kCSoft; }

// sanity before anything is sized from the record: alignments to a CCS read span at most a few hundred kilobases
int check_plausible(const BamRecord& rec) {
  uint64_t cols = 0;
  for (uint32_t c : rec.cigar) cols += c >> 4;
  if (cols > (1u << 24) || rec.pos < 0 || rec.pos > (1 << 24))
    return pfail(DCB_ERR_INVALID, "%s: implausible alignment (cigar / position)", rec.qname.c_str());
  return DCB_OK;
}

// Alignment columns [qs, qe) that survive the soft clips, out of `aln`
struct Clip { size_t aln = 0, qs = 0, qe = 0; };

// Every check expand_clip_indent makes on a subread once trim_insertions has run, from the trimmed cigar and the
// trimmed lengths of its sequence and kinetics alone, so that the host construction and the raw-record export refuse
// the same records with the same messages.  Fills the clip and the four sn values.
int check_trimmed(const BamRecord& rec, const std::vector<uint32_t>& cigar, size_t seq_len, size_t n_pw, size_t n_ip,
                  Clip* clip, float* sn) {
  size_t aln = 0, nq = 0, cig_cols = 0;
  bool any_soft = false;
  for (uint32_t c : cigar) {
    const int op = c & 15;
    const size_t len = c >> 4;
    if (op_has_column(op)) aln += len;
    if (op_has_query(op)) nq += len;
    if (op != kCHard) cig_cols += len;
    any_soft |= op == kCSoft && len;
  }
  if (nq != seq_len) return pfail(DCB_ERR_INVALID, "%s: cigar covers %zu query bases, sequence has %zu", rec.qname.c_str(), nq, seq_len);
  if (n_pw != nq || n_ip != nq) return pfail(DCB_ERR_INVALID, "%s: pw / ip tags do not match the sequence length", rec.qname.c_str());
  Tag t;
  if (!rec.find("sn", &t) || t.type != 'B' || t.count < 4) return pfail(DCB_ERR_INVALID, "%s: no sn tag", rec.qname.c_str());
  for (int i = 0; i < 4; ++i) sn[i] = (float)BamRecord::element(t, i);
  if (cig_cols != aln) return pfail(DCB_ERR_INVALID, "%s: unsupported cigar operation (pad)", rec.qname.c_str());
  clip->aln = aln; clip->qs = 0; clip->qe = aln;
  if (!any_soft) return DCB_OK;
  // query_alignment_start / _end: query bases outside leading / trailing soft clips
  size_t lead_soft = 0, trail_soft = 0;
  size_t i = 0;
  while (i < cigar.size() && (cigar[i] & 15) == kCHard) ++i;
  if (i < cigar.size() && (cigar[i] & 15) == kCSoft) lead_soft = cigar[i] >> 4;
  size_t j = cigar.size();
  while (j > 0 && (cigar[j - 1] & 15) == kCHard) --j;
  if (j > 0 && (cigar[j - 1] & 15) == kCSoft && j - 1 != i) trail_soft = cigar[j - 1] >> 4;
  // the alignment column of a query index
  auto column_of = [&](int64_t q, size_t* col) {
    if (q < 0) return false;
    size_t c0 = 0, q0 = 0;
    for (uint32_t c : cigar) {
      const int op = c & 15;
      const size_t len = c >> 4;
      if (op_has_query(op)) {
        if ((size_t)q < q0 + len) { *col = c0 + ((size_t)q - q0); return true; }
        q0 += len;
      }
      if (op_has_column(op)) c0 += len;
    }
    return false;
  };
  size_t last = 0;
  const bool f1 = column_of((int64_t)lead_soft, &clip->qs);
  const bool f2 = column_of((int64_t)seq_len - (int64_t)trail_soft - 1, &last);
  clip->qe = last + 1;
  if (!f1 || !f2 || clip->qe < clip->qs) return pfail(DCB_ERR_INVALID, "%s: cannot locate the aligned part", rec.qname.c_str());
  return DCB_OK;
}

int expand_clip_indent(BamRecord* rec, int ins_trim, Read* out) {
  std::vector<double> pw, ip;
  load_kinetics(*rec, &pw, &ip);
  if (int rc = check_plausible(*rec)) return rc;
  trim_insertions(rec, &pw, &ip, ins_trim);
  Clip clip;
  if (int rc = check_trimmed(*rec, rec->cigar, rec->seq.size(), pw.size(), ip.size(), &clip, out->sn)) return rc;
  std::vector<int32_t> read_idx, ccs_idx;
  aligned_pairs(rec->cigar, rec->pos, &read_idx, &ccs_idx);
  const size_t aln = read_idx.size();
  std::vector<char> seq(aln, kGap);
  std::vector<uint8_t> npw(aln, 0), nip(aln, 0);
  const bool rev = rec->flag & 16;
  if (rev) { std::reverse(pw.begin(), pw.end()); std::reverse(ip.begin(), ip.end()); }
  {
    size_t k = 0;
    for (size_t i = 0; i < aln; ++i)
      if (read_idx[i] >= 0) { seq[i] = rec->seq[k]; npw[i] = kinetic_u8(pw[k]); nip[i] = kinetic_u8(ip[k]); ++k; }
  }
  std::vector<uint8_t> cig;
  for (size_t ci = 0; ci < rec->cigar.size(); ++ci) {
    const int op = rec->cigar[ci] & 15;
    const size_t len = rec->cigar[ci] >> 4;
    if (op != kCHard) cig.insert(cig.end(), len, (uint8_t)op);
  }
  for (size_t i = 0; i < aln; ++i) if (cig[i] == kCSoft) seq[i] = kGap;
  const size_t qs = clip.qs, qe = clip.qe;
  const size_t indent = rec->pos > 0 ? (size_t)rec->pos : 0;
  const size_t n = indent + (qe - qs);
  out->name = rec->qname;
  out->bases.assign(n, kGap);
  out->cigar.assign(n, kCRefSkip);
  out->pw.assign(n, 0);
  out->ip.assign(n, 0);
  out->ccs_idx.assign(n, -1);
  for (size_t i = qs; i < qe; ++i) {
    const size_t o = indent + (i - qs);
    out->bases[o] = seq[i]; out->cigar[o] = cig[i]; out->pw[o] = npw[i]; out->ip[o] = nip[i]; out->ccs_idx[o] = ccs_idx[i];
  }
  out->strand = rev ? 2 : 1;
  return DCB_OK;
}

void construct_ccs_read(const BamRecord& rec, Read* out) {
  const size_t n = rec.seq.size();
  out->name = rec.qname;
  out->bases.assign(rec.seq.begin(), rec.seq.end());
  out->cigar.assign(n, kCMatch);
  out->pw.assign(n, 0);
  out->ip.assign(n, 0);
  out->strand = 0;
  out->ccs_idx.resize(n);
  out->bq.resize(n);
  out->bq_any = false;
  for (size_t i = 0; i < n; ++i) { out->ccs_idx[i] = (int32_t)i; out->bq[i] = rec.qual[i]; out->bq_any |= rec.qual[i] != 0; }
}

// space_out_subreads (pre_lib.py:1242-1276) for inference reads (no label)
void space_out(std::vector<Read>& reads) {
  for (Read& r : reads) { r.seq_indices.assign(r.bases.size(), 0); r.idx_seq = 0; r.idx_spaced = 0; r.done = false; }
  auto next_is_ins = [](const Read& r) { return r.idx_seq < r.cigar.size() && r.cigar[r.idx_seq] == kCIns; };
  for (;;) {
    bool all_done = true;
    for (const Read& r : reads) all_done &= r.done;
    if (all_done) break;
    bool any_ins = false;
    for (const Read& r : reads) {
      if (r.done) continue;
      if (next_is_ins(r)) { any_ins = true; break; }
    }
    for (Read& r : reads) {
      if (r.done) continue;
      if (any_ins && !next_is_ins(r)) {
        ++r.idx_spaced;                                        // add_gap
      } else {
        if (r.idx_seq < r.bases.size()) { r.seq_indices[r.idx_seq] = r.idx_spaced; ++r.idx_seq; ++r.idx_spaced; }   // move
        if (r.idx_seq >= r.bases.size()) r.done = true;
      }
    }
  }
  int32_t max_len = 0;
  for (const Read& r : reads) max_len = std::max(max_len, r.idx_spaced);
  for (Read& r : reads) {                                      // put_spacing
    std::vector<char> b(max_len, kGap);
    std::vector<uint8_t> pw(max_len, 0), ip(max_len, 0);
    std::vector<int32_t> ci(max_len, -1), bq;
    if (r.bq_any) bq.assign(max_len, -1);
    for (size_t i = 0; i < r.bases.size(); ++i) {
      const int32_t o = r.seq_indices[i];
      b[o] = r.bases[i]; pw[o] = r.pw[i]; ip[o] = r.ip[i]; ci[o] = r.ccs_idx[i];
      if (r.bq_any) bq[o] = r.bq[i];
    }
    r.bases.swap(b); r.pw.swap(pw); r.ip.swap(ip); r.ccs_idx.swap(ci);
    if (r.bq_any) r.bq.swap(bq);
  }
}

inline float encode_base(char c) {          // dc_constants.SEQ_VOCAB = ' ATCG'
  switch (c) { case 'A': return 1.f; case 'T': return 2.f; case 'C': return 3.f; case 'G': return 4.f; default: return 0.f; }
}

// One ZMW's records before any construction, in the flat arrays of dcb_prep_get_records (include/dcb200.h)
struct RawRecords {
  std::vector<int32_t> meta;      // [n_subreads][DCB_READ_META]
  std::vector<float> sn;          // [n_subreads][4]
  std::vector<uint32_t> cigar;
  std::vector<uint8_t> bases, pw, ip, ccs_bases, ccs_bq;
  std::vector<int32_t> wl;        // the `wl` tag, with smart windows
  int32_t ccs_bq_any = 0;
};

// Everything derived from one ZMW (what a DcExample holds after space_out_subreads + the window list)
struct ZmwState {
  std::vector<Read> reads;        // subreads..., ccs (spaced)
  std::string name, rg;
  float ec = 0, rq = 0;
  int has_ec = 0, has_np = 0, has_rq = 0, has_rg = 0;
  int32_t np_passes = 0, n_subreads = 0, ccs_length = 0;
  std::vector<int32_t> win_start; // column of every emitted window
  std::vector<int32_t> win_width; // its spaced width (overflow when > max_length)
  RawRecords raw;                 // raw-record mode (dcb_prep_export_records): the records instead of `reads`
  int label_status = -1;          // with a truth alignment open: DCB_LABEL_* of the fetch, the record in `label`
  BamRecord label;
  int label_rc = -1;              // label_of of `label` once dcb_prep_get_label asked for it (-1: not yet)
  std::string label_error;
  std::vector<uint32_t> label_cigar;
  std::vector<uint8_t> label_bases;
  int32_t label_info[DCB_LABEL_INFO] = {};
  int rc = DCB_OK;                // error of the processing step (message in `error`)
  std::string error;
};

struct ZmwJob {
  std::vector<BamRecord> group;
  BamRecord ccs;
  std::string name;
  int label_status = -1;
  BamRecord label;
};

// The part of a BAM index (.bai, SAM/BAM spec v1.6 section 5.2) a fetch needs: per reference, the smallest virtual
// offset any of its bins' chunks starts at (UINT64_MAX: the reference has no records) and, when `linear` is given, the
// linear index: per 16 kb window, the smallest virtual offset of a record that overlaps it (0: none recorded).
int read_bai(const std::string& path, size_t n_ref, std::vector<uint64_t>* first,
             std::vector<std::vector<uint64_t>>* linear = nullptr) {
  FILE* f = fopen(path.c_str(), "rb");
  if (!f) return pfail(DCB_ERR_INVALID, "cannot open the index %s (the truth alignment must be indexed)", path.c_str());
  std::vector<uint8_t> d;
  uint8_t buf[1 << 16];
  size_t n;
  while ((n = fread(buf, 1, sizeof buf, f)) > 0) d.insert(d.end(), buf, buf + n);
  fclose(f);
  size_t o = 0;
  bool bad = false;
  auto get = [&](void* dst, size_t bytes) { if (o + bytes > d.size()) { bad = true; return; } memcpy(dst, &d[o], bytes); o += bytes; };
  char magic[4] = {0, 0, 0, 0};
  int32_t nr = 0;
  get(magic, 4);
  get(&nr, 4);
  if (bad || memcmp(magic, "BAI\1", 4) || nr < 0 || (size_t)nr != n_ref)
    return pfail(DCB_ERR_INVALID, "%s: not a BAM index for this BAM", path.c_str());
  first->assign(n_ref, UINT64_MAX);
  if (linear) linear->clear();
  for (int32_t r = 0; r < nr && !bad; ++r) {
    int32_t n_bin = 0;
    get(&n_bin, 4);
    for (int32_t b = 0; b < n_bin && !bad; ++b) {
      uint32_t bin = 0;
      int32_t n_chunk = 0;
      get(&bin, 4);
      get(&n_chunk, 4);
      if (n_chunk < 0) bad = true;
      for (int32_t c = 0; c < n_chunk && !bad; ++c) {
        uint64_t beg = 0, end = 0;
        get(&beg, 8);
        get(&end, 8);
        if (bin != 37450) (*first)[r] = std::min((*first)[r], beg);   // 37450: the pseudo-bin of per-reference counts
      }
    }
    int32_t n_intv = 0;
    get(&n_intv, 4);
    if (n_intv < 0 || o + 8ull * n_intv > d.size()) { bad = true; break; }
    if (linear) linear->emplace_back((size_t)n_intv);
    if (linear && n_intv) memcpy(linear->back().data(), &d[o], 8ull * n_intv);
    o += 8ull * n_intv;
  }
  if (bad) return pfail(DCB_ERR_INVALID, "%s: truncated BAM index", path.c_str());
  return DCB_OK;
}

// The label record in the shape dcb_prep_get_label hands out: what expand_clip_indent keeps of it with truth_range set
// (pre_lib.py:1128-1239; no ins_trim).  Hard clips give no column; with any soft clip, the columns outside
// [query_alignment_start, query_alignment_end) go -- the soft clips and the deletions between them and the first / last
// aligned base.  info: DCB_LABEL_INFO entries.
int label_of(const BamRecord& rec, std::vector<uint32_t>* cigar, std::vector<uint8_t>* bases, int32_t* info) {
  const char* nm = rec.qname.c_str();
  if (rec.flag & 4) return pfail(DCB_ERR_INVALID, "%s: the truth alignment is unmapped", nm);
  if (int rc = check_plausible(rec)) return rc;
  std::vector<uint32_t> ops;
  for (uint32_t c : rec.cigar) {
    const int op = c & 15;
    if (op == kCHard || (c >> 4) == 0) continue;
    if (op != kCMatch && op != kCIns && op != kCDel && op != kCSoft && op != kCEq && op != kCDiff)
      return pfail(DCB_ERR_INVALID, "%s: truth alignment with a reference skip, pad or unknown cigar operation (not supported)", nm);
    ops.push_back(c);
  }
  size_t nq = 0;
  for (uint32_t c : ops) nq += op_has_query(c & 15) ? c >> 4 : 0;
  if (nq != rec.seq.size()) return pfail(DCB_ERR_INVALID, "%s: cigar covers %zu query bases, sequence has %zu", nm, nq, rec.seq.size());
  int32_t lead = 0, trail = 0;
  size_t a = 0, b = ops.size();
  if (a < b && (ops[a] & 15) == kCSoft) lead = (int32_t)(ops[a++] >> 4);
  if (a < b && (ops[b - 1] & 15) == kCSoft) trail = (int32_t)(ops[--b] >> 4);
  for (size_t i = a; i < b; ++i)
    if ((ops[i] & 15) == kCSoft) return pfail(DCB_ERR_INVALID, "%s: soft clip inside the truth alignment", nm);
  int32_t dropped = 0;
  if (lead || trail) {
    size_t i = a, j = b;
    while (i < j && (ops[i] & 15) == kCDel) dropped += (int32_t)(ops[i++] >> 4);
    while (j > i && (ops[j - 1] & 15) == kCDel) --j;
    if (i == j) return pfail(DCB_ERR_INVALID, "%s: cannot locate the aligned part", nm);
    a = i; b = j;
  }
  cigar->assign(ops.begin() + a, ops.begin() + b);
  bases->clear();
  size_t q = lead;
  for (uint32_t c : *cigar) {
    if (!op_has_query(c & 15)) continue;
    for (size_t k = 0; k < (c >> 4); ++k) {
      const char ch = rec.seq[q++];
      const uint8_t id = (uint8_t)encode_base(ch);
      if (!id) return pfail(DCB_ERR_INVALID, "%s: truth base '%c' outside ACGT (not supported)", nm, ch);
      bases->push_back(id);
    }
  }
  info[0] = DCB_LABEL_FOUND; info[1] = (int32_t)cigar->size(); info[2] = (int32_t)bases->size(); info[3] = rec.pos;
  info[4] = rec.pos + dropped; info[5] = lead; info[6] = trail; info[7] = rec.flag;
  return DCB_OK;
}

struct PrepCfg { int P = 0, L = 0, bq = 0, ins_trim = 0, R = 0; bool records = false, smart = false; dcb::PackedLayout pl{}; };

// What trim_insertions would leave of a record, without building it: the trimmed cigar and the lengths of the trimmed
// sequence and kinetics.  Follows trim_insertions to the letter: every operation but a deletion advances the sequence
// position, substrings and the kinetics mask are cut at the end of the sequence, and the mask is read from the far end
// for reverse-strand reads.
void trimmed_shape(const BamRecord& r, size_t n_pw, size_t n_ip, int ins_trim, std::vector<uint32_t>* cig, size_t* seq_len,
                   size_t* n_pw_out, size_t* n_ip_out) {
  if (ins_trim <= 0) { *cig = r.cigar; *seq_len = r.seq.size(); *n_pw_out = n_pw; *n_ip_out = n_ip; return; }
  const size_t n = r.seq.size();
  std::vector<std::pair<size_t, size_t>> cut;   // masked [begin, end) of the sequence, ascending and disjoint
  size_t sp = 0, kept = 0;
  cig->clear();
  for (uint32_t c : r.cigar) {
    const int op = c & 15;
    const size_t len = c >> 4;
    if (op == kCIns && (int)len > ins_trim) {
      if (sp < n) cut.emplace_back(sp, std::min(sp + len, n));
      sp += len;
    } else {
      cig->push_back(c);
      if (op != kCDel) { kept += std::min(len, n - std::min(sp, n)); sp += len; }
    }
  }
  *seq_len = kept;
  const bool rev = r.flag & 16;
  auto filtered = [&](size_t nv) {
    if (nv == 0) return (size_t)0;
    const size_t m = std::min(nv, n), lo = rev ? n - m : 0, hi = rev ? n : m;   // the mask positions the tag reaches
    size_t left = m;
    for (const auto& iv : cut) {
      const size_t a = std::max(iv.first, lo), b = std::min(iv.second, hi);
      if (b > a) left -= b - a;
    }
    return left;
  };
  *n_pw_out = filtered(n_pw);
  *n_ip_out = filtered(n_ip);
}

// Raw-record mode of process_zmw's per-subread step: the checks of expand_clip_indent, then the record as it is, with
// the clip the checks located.  Nothing is written for a record that fails.
int export_subread(const BamRecord& rec, int ins_trim, RawRecords* out) {
  std::vector<double> pw, ip;
  load_kinetics(rec, &pw, &ip);
  if (int rc = check_plausible(rec)) return rc;
  std::vector<uint32_t> cig;
  size_t seq_len, n_pw, n_ip;
  trimmed_shape(rec, pw.size(), ip.size(), ins_trim, &cig, &seq_len, &n_pw, &n_ip);
  Clip clip;
  float sn[4];
  if (int rc = check_trimmed(rec, cig, seq_len, n_pw, n_ip, &clip, sn)) return rc;
  // the construction kernels read the cigar as the SAM specification defines it; trim_insertions treats hard clips and
  // reference skips as if they held query bases, which only a record without them is unaffected by
  int64_t n_ins = 0;
  for (uint32_t c : cig) {
    const int op = c & 15;
    if (op == kCHard || op == kCRefSkip)
      return pfail(DCB_ERR_INVALID, "%s: hard clips / reference skips are not supported by the raw-record export", rec.qname.c_str());
    if (op == kCIns) n_ins += c >> 4;
  }
  const size_t n = rec.seq.size();
  const int32_t m[DCB_READ_META] = {(int32_t)out->cigar.size(), (int32_t)rec.cigar.size(), (int32_t)out->bases.size(), (int32_t)n,
                                    rec.pos, (rec.flag & 16) ? 1 : 0, (int32_t)clip.qs, (int32_t)clip.qe, (int32_t)n_ins, 0};
  out->meta.insert(out->meta.end(), m, m + DCB_READ_META);
  out->sn.insert(out->sn.end(), sn, sn + 4);
  out->cigar.insert(out->cigar.end(), rec.cigar.begin(), rec.cigar.end());
  for (size_t i = 0; i < n; ++i) {
    out->bases.push_back((uint8_t)encode_base(rec.seq[i]));
    out->pw.push_back(i < pw.size() ? kinetic_u8(pw[i]) : 0);
    out->ip.push_back(i < ip.size() ? kinetic_u8(ip[i]) : 0);
  }
  return DCB_OK;
}

// The `wl` tag of a CCS record (`--use_ccs_smart_windows`, pre_lib.py:1329-1331): CCS bases per window.  The reference
// fails on a missing tag, on a negative entry and on widths that do not add up to the CCS length; so does this.
int window_lengths(const BamRecord& c, const std::string& name, std::vector<int64_t>* wl) {
  Tag t;
  if (!c.find("wl", &t)) return pfail(DCB_ERR_INVALID, "%s: no wl tag (needed by --use_ccs_smart_windows)", name.c_str());
  if (t.type != 'B' || !strchr("cCsSiI", t.sub) || !t.sub)
    return pfail(DCB_ERR_INVALID, "%s: the wl tag is not an integer array", name.c_str());
  int64_t sum = 0;
  wl->resize(t.count);
  for (size_t j = 0; j < t.count; ++j) {
    (*wl)[j] = (int64_t)BamRecord::element(t, j);
    if ((*wl)[j] < 0) return pfail(DCB_ERR_INVALID, "%s: negative window length in the wl tag", name.c_str());
    sum += (*wl)[j];
  }
  if (sum != (int64_t)c.seq.size())
    return pfail(DCB_ERR_INVALID, "%s: the wl tag covers %lld CCS bases, the CCS read has %zu", name.c_str(), (long long)sum,
                 c.seq.size());
  return DCB_OK;
}

// DcExample.calculate_windows with window_widths (pre_lib.py:625-650) in closed form: window j holds the CCS bases
// [S, S + wl[j]) with S = wl[0] + ... + wl[j-1], plus the gap columns before the last of them, i.e. the spaced columns
// [col(S - 1) + 1, col(S + wl[j] - 1) + 1) where col(k) is the column of CCS base k (0 for S = 0).  An entry of 0 gives
// an empty window, which iter_examples drops (n_examples_no_ccs_idx).  Requires sum(wl) == CCS length.
void smart_windows(const Read& ccs, const std::vector<int64_t>& wl, std::vector<int32_t>* start, std::vector<int32_t>* width) {
  std::vector<int32_t> col;
  for (size_t i = 0; i < ccs.ccs_idx.size(); ++i)
    if (ccs.ccs_idx[i] >= 0) col.push_back((int32_t)i);
  int64_t s = 0;
  for (int64_t w : wl) {
    if (w == 0) continue;
    const int32_t a = s ? col[s - 1] + 1 : 0, b = col[s + w - 1] + 1;
    start->push_back(a);
    width->push_back(b - a);
    s += w;
  }
}

// CPU-heavy part, no I/O: expand_clip_indent per subread, construct_ccs_read, space_out_subreads, window list
void process_zmw(const PrepCfg& cfg, ZmwJob* job, ZmwState* st) {
  st->name = job->name;
  st->n_subreads = (int32_t)job->group.size();
  st->reads.clear();
  st->label_status = job->label_status;
  st->label = std::move(job->label);
  const BamRecord& c = job->ccs;
  if (cfg.records) {
    for (const BamRecord& r : job->group) {
      const int rc = export_subread(r, cfg.ins_trim, &st->raw);
      if (rc) { st->rc = rc; st->error = g_prep_error; st->raw = RawRecords(); return; }
    }
    for (size_t i = 0; i < c.seq.size(); ++i) {
      st->raw.ccs_bases.push_back((uint8_t)encode_base(c.seq[i]));
      st->raw.ccs_bq.push_back(c.qual[i]);
      st->raw.ccs_bq_any |= c.qual[i] != 0;
    }
  } else {
    st->reads.resize(job->group.size() + 1);
    for (size_t i = 0; i < job->group.size(); ++i) {
      const int rc = expand_clip_indent(&job->group[i], cfg.ins_trim, &st->reads[i]);
      if (rc) { st->rc = rc; st->error = g_prep_error; return; }
    }
    construct_ccs_read(c, &st->reads.back());
  }
  Tag t;
  st->has_ec = c.find("ec", &t); if (st->has_ec) st->ec = (float)BamRecord::scalar(t);
  st->has_np = c.find("np", &t); if (st->has_np) st->np_passes = (int32_t)BamRecord::scalar(t);
  st->has_rq = c.find("rq", &t); if (st->has_rq) st->rq = (float)BamRecord::scalar(t);
  st->has_rg = c.find("RG", &t) && t.type == 'Z'; if (st->has_rg) st->rg = reinterpret_cast<const char*>(t.p);
  st->ccs_length = (int32_t)c.seq.size();
  std::vector<int64_t> wl;
  if (cfg.smart) {
    const int rc = window_lengths(c, job->name, &wl);
    if (rc) { st->rc = rc; st->error = g_prep_error; st->raw = RawRecords(); return; }
    if (cfg.records) st->raw.wl.assign(wl.begin(), wl.end());   // each entry <= the CCS length: fits
  }
  if (cfg.records) return;
  space_out(st->reads);
  const Read& ccs = st->reads.back();
  const int width = (int)ccs.bases.size();
  st->win_start.clear();
  st->win_width.clear();
  if (cfg.smart) {
    smart_windows(ccs, wl, &st->win_start, &st->win_width);
    for (int32_t w : st->win_width)
      if (w > cfg.L && !ccs.bq_any) {
        st->rc = pfail(DCB_ERR_INVALID, "%s: overflow window in a CCS read without base qualities (not supported)", job->name.c_str());
        st->error = g_prep_error;
        return;
      }
    return;
  }
  // DcExample.iter_examples (pre_lib.py:625-697), fixed-width windows
  int ccs_width = width;
  while (ccs_width > 0 && (ccs.bases[ccs_width - 1] == ' ' || ccs.bases[ccs_width - 1] == '\t' || ccs.bases[ccs_width - 1] == '\n')) --ccs_width;
  const int nwin = (ccs_width + cfg.L - 1) / cfg.L;
  int start = 0;
  for (int w = 0; w < nwin; ++w) {
    if (start > ccs_width) break;
    const int s0 = start;
    start += cfg.L;
    bool any = false;
    for (int i = s0; i < std::min(s0 + cfg.L, width); ++i) any |= ccs.ccs_idx[i] >= 0;
    if (!any) continue;                                         // n_examples_no_ccs_idx
    st->win_start.push_back(s0);
    st->win_width.push_back(std::min(cfg.L, width - s0));
  }
}

}  // namespace

struct dcb_prep {
  BamReader sub, ccs;
  PrepCfg cfg;
  // dcb_prep_open_truth: the truth alignment, its references by name and each one's first virtual offset (read_bai)
  BamReader truth;
  bool have_truth = false;
  std::map<std::string, int32_t> truth_tid;
  std::vector<uint64_t> truth_first;
  bool have_pending = false, sub_eof = false;
  BamRecord pending;
  int64_t pending_zm = 0;
  ZmwState cur;                   // the ZMW handed out by the last dcb_prep_next_zmw
  // optional worker pool (dcb_prep_set_threads): one reader thread decodes and groups, n workers process, results are
  // handed out in file order
  int n_threads = 0;
  bool started = false, stop = false;
  std::thread reader;
  std::vector<std::thread> workers;
  std::mutex mu;
  std::condition_variable cv_job, cv_res, cv_space;
  std::deque<std::pair<int64_t, ZmwJob>> jobs;
  std::map<int64_t, ZmwState> results;
  int64_t next_seq = 0, total = -1;   // total: number of ZMWs once the reader hit the end (or an error)
  int reader_rc = DCB_OK;
  std::string reader_error;
};

namespace {

// next(truth_to_ccs.fetch(name)) (pre_lib.py:1001-1014): the first record of the reference named after the CCS read, found
// by seeking to the smallest chunk start of its bins and reading on to the first record with its tid; none when the
// reference is not in the header or has no records.  A supplementary first record is reported as such.
int fetch_label(dcb_prep* p, ZmwJob* job) {
  job->label_status = DCB_LABEL_NOT_FOUND;
  auto it = p->truth_tid.find(job->name);
  if (it == p->truth_tid.end() || p->truth_first[it->second] == UINT64_MAX) return 1;
  if (!p->truth.z.seek(p->truth_first[it->second])) return pfail(DCB_ERR_INVALID, "truth alignment: bad index offset for %s", job->name.c_str());
  for (;;) {
    const int rc = p->truth.next(&job->label);
    if (rc < 0) return rc;
    if (rc == 0 || job->label.refid < 0 || job->label.refid > it->second) return 1;
    if (job->label.refid == it->second) break;
  }
  job->label_status = (job->label.flag & 0x800) ? DCB_LABEL_SUPPLEMENTARY : DCB_LABEL_FOUND;
  return 1;
}

// Sequential I/O: the next group of mapped subreads with one zm (SubreadGrouper, pre_lib.py:50-91) and its CCS record
// (pre_lib.py:1322-1330).  1 = job filled, 0 = end of file, < 0 = error.
int read_job(dcb_prep* p, ZmwJob* job) {
  std::vector<BamRecord>& group = job->group;
  group.clear();
  int64_t zm = 0;
  bool have_zm = false;
  auto zm_of = [&](const BamRecord& r, int64_t* v) {
    Tag t;
    if (!r.find("zm", &t)) return false;
    *v = (int64_t)BamRecord::scalar(t);
    return true;
  };
  // consecutive records with the same zm; unmapped records are dropped, but the very first record of the file sets the
  // first group's zm even when it is unmapped
  if (p->have_pending) { group.push_back(p->pending); zm = p->pending_zm; have_zm = true; p->have_pending = false; }
  while (!p->sub_eof) {
    BamRecord r;
    const int rc = p->sub.next(&r);
    if (rc < 0) return rc;
    if (rc == 0) { p->sub_eof = true; break; }
    int64_t rz;
    if (!zm_of(r, &rz)) return pfail(DCB_ERR_INVALID, "%s: no zm tag", r.qname.c_str());
    if (!have_zm) { zm = rz; have_zm = true; if (!(r.flag & 4)) group.push_back(r); continue; }
    if (r.flag & 4) continue;
    if (rz == zm) { group.push_back(r); continue; }
    if (!group.empty()) { p->pending = r; p->pending_zm = rz; p->have_pending = true; break; }
    group.push_back(r); zm = rz;
  }
  if (group.empty()) return 0;
  const int32_t refid = group[0].refid;
  if (refid < 0 || refid >= (int32_t)p->sub.refs.size()) return pfail(DCB_ERR_INVALID, "%s: no reference name", group[0].qname.c_str());
  job->name = p->sub.refs[refid];
  for (;;) {
    const int rc = p->ccs.next(&job->ccs);
    if (rc < 0) return rc;
    if (rc == 0) return pfail(DCB_ERR_INVALID, "ccs bam does not contain %s", job->name.c_str());
    if (job->ccs.qname == job->name) break;
  }
  return p->have_truth ? fetch_label(p, job) : 1;
}

void reader_main(dcb_prep* p) {
  int64_t seq = 0;
  for (;;) {
    ZmwJob job;
    const int rc = read_job(p, &job);
    std::unique_lock<std::mutex> lk(p->mu);
    if (rc <= 0) {
      if (rc < 0) { p->reader_rc = rc; p->reader_error = g_prep_error; }
      p->total = seq;
      p->cv_job.notify_all();
      p->cv_res.notify_all();
      return;
    }
    p->cv_space.wait(lk, [&] { return p->stop || (int64_t)(p->jobs.size() + p->results.size()) < 4ll * p->n_threads + 4; });
    if (p->stop) return;
    p->jobs.emplace_back(seq++, std::move(job));
    p->cv_job.notify_one();
  }
}

void worker_main(dcb_prep* p) {
  for (;;) {
    std::pair<int64_t, ZmwJob> item;
    {
      std::unique_lock<std::mutex> lk(p->mu);
      p->cv_job.wait(lk, [&] { return p->stop || !p->jobs.empty() || p->total >= 0; });
      if (p->stop) return;
      if (p->jobs.empty()) return;                 // reader finished and nothing left
      item = std::move(p->jobs.front());
      p->jobs.pop_front();
    }
    ZmwState st;
    process_zmw(p->cfg, &item.second, &st);
    {
      std::lock_guard<std::mutex> lk(p->mu);
      p->results.emplace(item.first, std::move(st));
    }
    p->cv_res.notify_all();
  }
}

void stop_threads(dcb_prep* p) {
  if (!p->started) return;
  {
    std::lock_guard<std::mutex> lk(p->mu);
    p->stop = true;
  }
  p->cv_job.notify_all(); p->cv_res.notify_all(); p->cv_space.notify_all();
  if (p->reader.joinable()) p->reader.join();
  for (auto& w : p->workers) if (w.joinable()) w.join();
  p->started = false;
}

}  // namespace

extern "C" {

const char* dcb_prep_last_error(void) { return g_prep_error.c_str(); }

int dcb_prep_open(const char* subreads_to_ccs_bam, const char* ccs_bam, int32_t max_passes, int32_t max_length,
                  int32_t use_ccs_bq, int32_t ins_trim, dcb_prep** out) {
  if (!subreads_to_ccs_bam || !ccs_bam || !out || max_passes <= 0 || max_length <= 0) return pfail(DCB_ERR_INVALID, "dcb_prep_open: bad argument");
  dcb_prep* p = new dcb_prep();
  PrepCfg& c = p->cfg;
  c.P = max_passes; c.L = max_length; c.bq = use_ccs_bq ? 1 : 0; c.ins_trim = ins_trim;
  c.R = 4 * max_passes + 5 + c.bq;
  c.pl = dcb::make_packed_layout(max_passes, max_length, c.bq);
  int rc = p->sub.open(subreads_to_ccs_bam);
  if (!rc) rc = p->ccs.open(ccs_bam);
  if (rc) { delete p; return rc; }
  *out = p;
  return DCB_OK;
}

// Process ZMWs on `n_threads` worker threads (plus one thread that decodes the BAMs); results still come out of
// dcb_prep_next_zmw in file order.  Call before the first dcb_prep_next_zmw; n_threads <= 0 keeps everything on the caller.
int dcb_prep_set_threads(dcb_prep* p, int32_t n_threads) {
  if (!p) return pfail(DCB_ERR_INVALID, "dcb_prep_set_threads: null handle");
  if (p->started || p->next_seq) return pfail(DCB_ERR_STATE, "dcb_prep_set_threads: the stream has already started");
  p->n_threads = n_threads > 0 ? std::min(n_threads, 256) : 0;
  return DCB_OK;
}

void dcb_prep_close(dcb_prep* p) {
  if (!p) return;
  stop_threads(p);
  delete p;
}

// Advances to the next ZMW that has mapped subreads.  Returns 1 and fills `info`, 0 at the end of the file, < 0 on error.
int dcb_prep_next_zmw(dcb_prep* p, dcb_zmw_info* info) {
  if (!p || !info) return pfail(DCB_ERR_INVALID, "dcb_prep_next_zmw: null argument");
  if (p->n_threads > 0) {
    if (!p->started) {
      p->started = true;
      p->reader = std::thread(reader_main, p);
      for (int i = 0; i < p->n_threads; ++i) p->workers.emplace_back(worker_main, p);
    }
    std::unique_lock<std::mutex> lk(p->mu);
    p->cv_res.wait(lk, [&] { return p->results.count(p->next_seq) || (p->total >= 0 && p->next_seq >= p->total); });
    auto it = p->results.find(p->next_seq);
    if (it == p->results.end()) {
      p->cur.raw = RawRecords();   // nothing to export after the end or an error
      if (p->reader_rc) { g_prep_error = p->reader_error; return p->reader_rc; }
      return 0;
    }
    p->cur = std::move(it->second);
    p->results.erase(it);
    ++p->next_seq;
    lk.unlock();
    p->cv_space.notify_all();
  } else {
    ZmwJob job;
    const int rc = read_job(p, &job);
    if (rc <= 0) { p->cur.raw = RawRecords(); return rc; }
    p->cur = ZmwState();
    process_zmw(p->cfg, &job, &p->cur);
    ++p->next_seq;
  }
  if (p->cur.rc) { g_prep_error = p->cur.error; return p->cur.rc; }
  const ZmwState& st = p->cur;
  memset(info, 0, sizeof *info);
  info->n_windows = (int32_t)st.win_start.size();
  info->n_subreads = st.n_subreads;
  info->name = st.name.c_str();
  info->has_ec = st.has_ec; info->ec = st.ec;
  info->has_np = st.has_np; info->np_num_passes = st.np_passes;
  info->has_rq = st.has_rq; info->rq = st.rq;
  info->rg = st.has_rg ? st.rg.c_str() : nullptr;
  info->ccs_length = st.ccs_length;
  info->spaced_width = st.reads.empty() ? 0 : (int32_t)st.reads.back().bases.size();
  return 1;
}

// The windows of the current ZMW (DcExample.extract_features / to_features_dict, pre_lib.py:704-762).  Every output may
// be NULL.  rows: float32 [n, R, L]; packed: [n, packed_window_bytes]; window_pos / num_passes: [n]; overflow: [n]
// (always 0 with fixed-width windows); ccs_bq: int16 [n, L] (-1 at gaps and padding).
int dcb_prep_get_windows(dcb_prep* p, float* rows, uint8_t* packed, int32_t* window_pos, uint8_t* overflow,
                         int16_t* ccs_bq, int32_t* num_passes) {
  if (!p) return pfail(DCB_ERR_INVALID, "dcb_prep_get_windows: null handle");
  const ZmwState& st = p->cur;
  if (st.reads.empty()) return pfail(DCB_ERR_STATE, "dcb_prep_get_windows: no ZMW loaded (or the stream is in raw-record mode)");
  const PrepCfg& cf = p->cfg;
  const int L = cf.L, P = cf.P, R = cf.R;
  const size_t nsub = st.reads.size() - 1;
  const int keep = (int)std::min<size_t>(P, nsub);
  const Read& ccs = st.reads.back();
  for (size_t w = 0; w < st.win_start.size(); ++w) {
    const int s = st.win_start[w];
    // columns present; the rest is padding.  An overflow window (width > L) is never scored: its rows hold its first L
    // columns, and dcb_prep_get_overflow_ccs hands out the full-width CCS that replaces it.
    const int n = std::min(L, st.win_width[w]);
    if (rows) {
      float* d = rows + w * (size_t)R * L;
      memset(d, 0, sizeof(float) * (size_t)R * L);
      for (int k = 0; k < keep; ++k) {
        const Read& r = st.reads[k];
        for (int i = 0; i < n; ++i) {
          d[(size_t)k * L + i] = encode_base(r.bases[s + i]);
          d[(size_t)(P + k) * L + i] = (float)r.pw[s + i];
          d[(size_t)(2 * P + k) * L + i] = (float)r.ip[s + i];
        }
        for (int i = 0; i < L; ++i) d[(size_t)(3 * P + k) * L + i] = (float)r.strand;   // repeated over the whole width
      }
      for (int i = 0; i < n; ++i) d[(size_t)4 * P * L + i] = encode_base(ccs.bases[s + i]);
      if (cf.bq)
        for (int i = 0; i < L; ++i) d[(size_t)(4 * P + 1) * L + i] = (i < n && ccs.bq_any) ? (float)ccs.bq[s + i] : -1.f;
      for (int j = 0; j < 4; ++j)
        for (int i = 0; i < L; ++i) d[(size_t)(R - 4 + j) * L + i] = st.reads[0].sn[j];
    }
    if (packed) {
      uint8_t* o = packed + w * (size_t)cf.pl.stride;
      memset(o, 0, cf.pl.stride);
      for (int k = 0; k < keep; ++k) {
        const Read& r = st.reads[k];
        for (int i = 0; i < L; ++i) {
          const int base = i < n ? (int)encode_base(r.bases[s + i]) : 0;
          o[k * L + i] = (uint8_t)(base | (r.strand << 3));
        }
        for (int i = 0; i < n; ++i) { o[(P + k) * L + i] = r.pw[s + i]; o[(2 * P + k) * L + i] = r.ip[s + i]; }
      }
      for (int i = 0; i < n; ++i) o[3 * P * L + i] = (uint8_t)encode_base(ccs.bases[s + i]);
      if (cf.bq)
        for (int i = 0; i < L; ++i) o[(3 * P + 1) * L + i] = (uint8_t)(((i < n && ccs.bq_any) ? ccs.bq[s + i] : -1) + 1);
      memcpy(o + cf.pl.sn_off, st.reads[0].sn, 16);
    }
    if (window_pos) {
      int32_t mn = 0;
      bool found = false;
      for (int i = 0; i < st.win_width[w]; ++i) {
        const int32_t v = ccs.ccs_idx[s + i];
        if (v >= 0 && (!found || v < mn)) { mn = v; found = true; }
      }
      window_pos[w] = mn;                                       // ccs_bounds.start
    }
    if (overflow) overflow[w] = st.win_width[w] > L;
    if (num_passes) num_passes[w] = keep;
    if (ccs_bq)
      for (int i = 0; i < L; ++i) ccs_bq[w * (size_t)L + i] = (int16_t)((i < n && ccs.bq_any) ? ccs.bq[s + i] : -1);
  }
  return DCB_OK;
}

// Windows cut at the CCS record's `wl` widths instead of every max_length columns.  Call before the first
// dcb_prep_next_zmw.  In raw-record mode the tag is checked and handed out (dcb_prep_get_window_lengths).
int dcb_prep_use_ccs_smart_windows(dcb_prep* p, int32_t enabled) {
  if (!p) return pfail(DCB_ERR_INVALID, "dcb_prep_use_ccs_smart_windows: null handle");
  if (p->started || p->next_seq) return pfail(DCB_ERR_STATE, "dcb_prep_use_ccs_smart_windows: the stream has already started");
  p->cfg.smart = enabled != 0;
  return DCB_OK;
}

// Raw-record mode with smart windows: the loaded ZMW's `wl` tag.
int dcb_prep_get_window_lengths(dcb_prep* p, int32_t* n, int32_t* wl) {
  if (!p || !n) return pfail(DCB_ERR_INVALID, "dcb_prep_get_window_lengths: null argument");
  if (!p->cfg.records || !p->cfg.smart || p->cur.raw.meta.empty())
    return pfail(DCB_ERR_STATE, "dcb_prep_get_window_lengths: no ZMW loaded in raw-record mode with smart windows");
  *n = (int32_t)p->cur.raw.wl.size();
  if (wl) std::copy(p->cur.raw.wl.begin(), p->cur.raw.wl.end(), wl);
  return DCB_OK;
}

// Spaced width of every window of the current ZMW, int32 [n_windows].
int dcb_prep_get_window_widths(dcb_prep* p, int32_t* width) {
  if (!p || !width) return pfail(DCB_ERR_INVALID, "dcb_prep_get_window_widths: null argument");
  if (p->cur.reads.empty()) return pfail(DCB_ERR_STATE, "dcb_prep_get_window_widths: no ZMW loaded (or the stream is in raw-record mode)");
  std::copy(p->cur.win_width.begin(), p->cur.win_width.end(), width);
  return DCB_OK;
}

// The CCS of every overflow window of the current ZMW over its full width, windows back to back in window order:
// ccs_ids u8 (0..4, ' ATCG') and ccs_bq int16 (-1 at gap columns), sum of the overflow windows' widths each.  These
// are the feature values to_features_dict gives such a window (it is neither padded nor truncated).  Either may be NULL.
int dcb_prep_get_overflow_ccs(dcb_prep* p, uint8_t* ccs_ids, int16_t* ccs_bq) {
  if (!p) return pfail(DCB_ERR_INVALID, "dcb_prep_get_overflow_ccs: null handle");
  const ZmwState& st = p->cur;
  if (st.reads.empty()) return pfail(DCB_ERR_STATE, "dcb_prep_get_overflow_ccs: no ZMW loaded (or the stream is in raw-record mode)");
  const Read& ccs = st.reads.back();
  size_t o = 0;
  for (size_t w = 0; w < st.win_start.size(); ++w) {
    if (st.win_width[w] <= p->cfg.L) continue;
    for (int i = 0; i < st.win_width[w]; ++i, ++o) {
      const int c = st.win_start[w] + i;
      if (ccs_ids) ccs_ids[o] = (uint8_t)encode_base(ccs.bases[c]);
      if (ccs_bq) ccs_bq[o] = (int16_t)ccs.bq[c];   // overflow windows only exist where bq_any (process_zmw)
    }
  }
  return DCB_OK;
}

// Raw-record mode: dcb_prep_next_zmw decodes, validates and keeps the records of each ZMW for dcb_prep_get_records and
// builds no windows (n_windows and spaced_width are 0).  Call before the first dcb_prep_next_zmw.
int dcb_prep_export_records(dcb_prep* p, int32_t enabled) {
  if (!p) return pfail(DCB_ERR_INVALID, "dcb_prep_export_records: null handle");
  if (p->started || p->next_seq) return pfail(DCB_ERR_STATE, "dcb_prep_export_records: the stream has already started");
  p->cfg.records = enabled != 0;
  return DCB_OK;
}

// The loaded ZMW's records.  sizes (always written): subreads, cigar operations, query bases, CCS length, whether any
// CCS base quality is non-zero.  Every array may be NULL (a first call with only `sizes` tells how to size them).
int dcb_prep_get_records(dcb_prep* p, int64_t* sizes, int32_t* read_meta, float* read_sn, uint32_t* cigar,
                         uint8_t* bases, uint8_t* pw, uint8_t* ip, uint8_t* ccs_bases, uint8_t* ccs_bq) {
  if (!p || !sizes) return pfail(DCB_ERR_INVALID, "dcb_prep_get_records: null argument");
  if (!p->cfg.records || p->cur.raw.meta.empty()) return pfail(DCB_ERR_STATE, "dcb_prep_get_records: no ZMW loaded in raw-record mode");
  const RawRecords& r = p->cur.raw;
  sizes[0] = (int64_t)(r.meta.size() / DCB_READ_META); sizes[1] = (int64_t)r.cigar.size(); sizes[2] = (int64_t)r.bases.size();
  sizes[3] = (int64_t)r.ccs_bases.size(); sizes[4] = r.ccs_bq_any;
  auto put = [](void* dst, const void* src, size_t bytes) { if (dst && bytes) memcpy(dst, src, bytes); };
  put(read_meta, r.meta.data(), r.meta.size() * 4); put(read_sn, r.sn.data(), r.sn.size() * 4);
  put(cigar, r.cigar.data(), r.cigar.size() * 4);
  put(bases, r.bases.data(), r.bases.size()); put(pw, r.pw.data(), r.pw.size()); put(ip, r.ip.data(), r.ip.size());
  put(ccs_bases, r.ccs_bases.data(), r.ccs_bases.size()); put(ccs_bq, r.ccs_bq.data(), r.ccs_bq.size());
  return DCB_OK;
}

// Training mode: open the truth alignment to the CCS reads and its index (path + ".bai").  Call before the first
// dcb_prep_next_zmw; every ZMW then fetches its label record on the decoding side.
int dcb_prep_open_truth(dcb_prep* p, const char* truth_to_ccs_bam) {
  if (!p || !truth_to_ccs_bam) return pfail(DCB_ERR_INVALID, "dcb_prep_open_truth: null argument");
  if (p->started || p->next_seq || p->have_truth) return pfail(DCB_ERR_STATE, "dcb_prep_open_truth: the stream has already started");
  if (int rc = p->truth.open(truth_to_ccs_bam)) return rc;
  if (int rc = read_bai(std::string(truth_to_ccs_bam) + ".bai", p->truth.refs.size(), &p->truth_first)) return rc;
  for (size_t i = 0; i < p->truth.refs.size(); ++i) p->truth_tid.emplace(p->truth.refs[i], (int32_t)i);
  p->have_truth = true;
  return DCB_OK;
}

// The loaded ZMW's label (include/dcb200.h).  info [DCB_LABEL_INFO] is always written; cigar / bases may be NULL.
int dcb_prep_get_label(dcb_prep* p, int32_t* info, uint32_t* cigar, uint8_t* bases) {
  if (!p || !info) return pfail(DCB_ERR_INVALID, "dcb_prep_get_label: null argument");
  memset(info, 0, sizeof(int32_t) * DCB_LABEL_INFO);
  if (!p->have_truth || p->cur.label_status < 0) return pfail(DCB_ERR_STATE, "dcb_prep_get_label: no ZMW loaded with a truth alignment open");
  ZmwState& st = p->cur;
  info[0] = st.label_status;
  if (st.label_status != DCB_LABEL_FOUND) return DCB_OK;
  if (st.label_rc < 0) {   // converted once per ZMW, on the first call
    st.label_rc = label_of(st.label, &st.label_cigar, &st.label_bases, st.label_info);
    if (st.label_rc) st.label_error = g_prep_error;
  }
  if (st.label_rc) { g_prep_error = st.label_error; return st.label_rc; }
  std::copy(st.label_info, st.label_info + DCB_LABEL_INFO, info);
  if (cigar) std::copy(st.label_cigar.begin(), st.label_cigar.end(), cigar);
  if (bases) std::copy(st.label_bases.begin(), st.label_bases.end(), bases);
  return DCB_OK;
}

// Header text of the CCS BAM (the output BAM reuses it, quick_inference.py:894-897).
const char* dcb_prep_ccs_header(dcb_prep* p) { return p ? p->ccs.header_text.c_str() : ""; }

}  // extern "C"

// ----------------------------------------------------------------------------------------------- BAM writer
struct dcb_bamw {
  FILE* f = nullptr;
  std::vector<uint8_t> buf;
  bool failed = false;
  void flush_block(bool force_empty = false) {
    if (buf.empty() && !force_empty) return;
    const uLong src = (uLong)buf.size();
    std::vector<uint8_t> comp(compressBound(src) + 64);
    z_stream zs;
    memset(&zs, 0, sizeof zs);
    if (deflateInit2(&zs, Z_DEFAULT_COMPRESSION, Z_DEFLATED, -15, 8, Z_DEFAULT_STRATEGY) != Z_OK) { failed = true; return; }
    zs.next_in = buf.data(); zs.avail_in = (uInt)src;
    zs.next_out = comp.data(); zs.avail_out = (uInt)comp.size();
    const int rc = deflate(&zs, Z_FINISH);
    const size_t clen = zs.total_out;
    deflateEnd(&zs);
    if (rc != Z_STREAM_END) { failed = true; return; }
    const uint32_t bsize = (uint32_t)(clen + 25);              // 18 header + data + 8 trailer - 1
    uint8_t h[18] = {31, 139, 8, 4, 0, 0, 0, 0, 0, 255, 6, 0, 'B', 'C', 2, 0, (uint8_t)(bsize & 255), (uint8_t)(bsize >> 8)};
    const uint32_t crc = (uint32_t)crc32(0, buf.data(), (uInt)src), isz = (uint32_t)src;
    uint8_t t[8] = {(uint8_t)crc, (uint8_t)(crc >> 8), (uint8_t)(crc >> 16), (uint8_t)(crc >> 24),
                    (uint8_t)isz, (uint8_t)(isz >> 8), (uint8_t)(isz >> 16), (uint8_t)(isz >> 24)};
    if (fwrite(h, 1, 18, f) != 18 || fwrite(comp.data(), 1, clen, f) != clen || fwrite(t, 1, 8, f) != 8) failed = true;
    buf.clear();
  }
  void put(const void* p, size_t n) {
    const uint8_t* s = static_cast<const uint8_t*>(p);
    while (n) {
      const size_t room = 0xff00 - buf.size();
      const size_t take = std::min(room, n);
      buf.insert(buf.end(), s, s + take);
      s += take; n -= take;
      if (buf.size() >= 0xff00) flush_block();
    }
  }
};

extern "C" {

int dcb_bamw_open(const char* path, const char* header_text, dcb_bamw** out) {
  if (!path || !out) return pfail(DCB_ERR_INVALID, "dcb_bamw_open: bad argument");
  dcb_bamw* w = new dcb_bamw();
  w->f = fopen(path, "wb");
  if (!w->f) { delete w; return pfail(DCB_ERR_INVALID, "cannot create %s", path); }
  const std::string text = header_text ? header_text : "";
  const int32_t l_text = (int32_t)text.size(), n_ref = 0;
  w->put("BAM\1", 4);
  w->put(&l_text, 4);
  w->put(text.data(), text.size());
  w->put(&n_ref, 4);
  w->flush_block();
  *out = w;
  return DCB_OK;
}

// One unaligned record as quick_inference.py:742-760 writes it: flag 4, mapq 255, tags ec:f (-1 when absent), np:i, rq:f,
// RG:Z, zm:i (the ZMW number parsed from the name "movie/zmw/ccs").
int dcb_bamw_write(dcb_bamw* w, const char* name, const uint8_t* seq, const uint8_t* qual_phred33, int32_t len, int32_t has_ec,
                   float ec, int32_t np_num_passes, float rq, const char* rg) {
  if (!w || !name || !seq || !qual_phred33 || len < 0) return pfail(DCB_ERR_INVALID, "dcb_bamw_write: bad argument");
  const size_t l_name = strlen(name) + 1;
  if (l_name > 255) return pfail(DCB_ERR_INVALID, "read name too long");
  int64_t zm = 0;
  {
    const char* a = strchr(name, '/');
    if (!a) return pfail(DCB_ERR_INVALID, "%s: cannot parse the ZMW number", name);
    zm = strtoll(a + 1, nullptr, 10);
  }
  std::vector<uint8_t> rec;
  auto put32 = [&](int32_t v) { const uint8_t* p = reinterpret_cast<const uint8_t*>(&v); rec.insert(rec.end(), p, p + 4); };
  put32(-1);                                                   // refID
  put32(-1);                                                   // pos
  rec.push_back((uint8_t)l_name);
  rec.push_back(255);                                          // mapq
  rec.push_back(4680 & 255); rec.push_back(4680 >> 8);         // bin of an unmapped read (reg2bin(-1, 0))
  rec.push_back(0); rec.push_back(0);                          // n_cigar_op
  rec.push_back(4); rec.push_back(0);                          // flag 4
  put32(len);
  put32(-1); put32(-1); put32(0);                              // next refID, next pos, tlen
  rec.insert(rec.end(), name, name + l_name);
  static int8_t code[256];
  static bool init = false;
  if (!init) { memset(code, 15, sizeof code); const char* nt = "=ACMGRSVTWYHKDBN"; for (int i = 0; i < 16; ++i) code[(uint8_t)nt[i]] = (int8_t)i; init = true; }
  for (int i = 0; i < len; i += 2) {
    const int hi = code[seq[i]], lo = i + 1 < len ? code[seq[i + 1]] : 0;
    rec.push_back((uint8_t)((hi << 4) | lo));
  }
  for (int i = 0; i < len; ++i) rec.push_back((uint8_t)(qual_phred33[i] - 33));
  auto tagf = [&](const char* n, float v) { rec.push_back(n[0]); rec.push_back(n[1]); rec.push_back('f'); const uint8_t* p = reinterpret_cast<const uint8_t*>(&v); rec.insert(rec.end(), p, p + 4); };
  auto tagi = [&](const char* n, int32_t v) { rec.push_back(n[0]); rec.push_back(n[1]); rec.push_back('i'); put32(v); };
  tagf("ec", (has_ec && ec != 0.f) ? ec : -1.f);               // `ec or -1`
  tagi("np", np_num_passes);
  tagf("rq", rq);
  if (rg) { rec.push_back('R'); rec.push_back('G'); rec.push_back('Z'); rec.insert(rec.end(), rg, rg + strlen(rg) + 1); }
  tagi("zm", (int32_t)zm);
  const int32_t bs = (int32_t)rec.size();
  w->put(&bs, 4);
  w->put(rec.data(), rec.size());
  return w->failed ? pfail(DCB_ERR_INVALID, "write failed") : DCB_OK;
}

int dcb_bamw_close(dcb_bamw* w) {
  if (!w) return DCB_OK;
  w->flush_block();
  w->flush_block(true);                                        // the BGZF end-of-file marker: an empty block
  const bool bad = w->failed || fclose(w->f) != 0;
  delete w;
  return bad ? pfail(DCB_ERR_INVALID, "closing the BAM failed") : DCB_OK;
}

}  // extern "C"

// ----------------------------------------------------------------------------------------------- calibration reader
// The host side of `calculate_baseq_calibration` (include/dcb200.h "base-quality calibration"): the reads an indexed,
// coordinate-sorted BAM holds over a reference span, filtered as get_quality_calibration_stats filters them, exported
// in batches as flat arrays for dcb_calib_count; and the reference's bases from a FASTA file through its .fai.
struct FaiEntry { std::string name; int64_t len = 0, off = 0, line_bases = 0, line_width = 0; };

struct dcb_calib {
  BamReader bam;
  std::vector<uint64_t> first;
  std::vector<std::vector<uint64_t>> linear;
  std::map<std::string, int32_t> tid;
  std::string bam_contigs, fasta_contigs;
  FILE* fa = nullptr;
  std::vector<FaiEntry> fai;
  int n_threads = 1;
  // the current query (dcb_calib_query)
  int32_t q_tid = -1;
  int64_t q_lo = 0, q_hi = 0, q_min_pos = 0;
  int q_min_mapq = 0;
  bool q_done = true;
  // the current batch: the kept records' bytes, then their export
  std::vector<uint8_t> arena;
  std::vector<size_t> rec_at;
  std::vector<int32_t> meta;
  std::vector<uint32_t> cigar;
  std::vector<uint8_t> seq, qual;
  std::vector<std::string> names;
  ~dcb_calib() { if (fa) fclose(fa); }
};

namespace {

// BAM flags get_quality_calibration_stats skips: duplicate, qcfail, secondary, unmapped, supplementary
constexpr uint16_t kCalibSkipFlags = 0x400 | 0x200 | 0x100 | 0x4 | 0x800;

// Reference length of a raw record's cigar (M, D, N, =, X)
int64_t raw_ref_len(const uint8_t* b) {
  uint16_t n_cig;
  memcpy(&n_cig, b + 12, 2);
  const uint8_t* c = b + 32 + b[8];
  int64_t n = 0;
  for (int k = 0; k < n_cig; ++k) {
    uint32_t v;
    memcpy(&v, c + 4 * k, 4);
    const int op = v & 15;
    if (op == kCMatch || op == kCDel || op == kCRefSkip || op == kCEq || op == kCDiff) n += v >> 4;
  }
  return n;
}

// samtools faidx's index, built in memory: per sequence its length, the offset of its first base, and the bases and
// bytes per line (every line but the last of a sequence has the same length).
int build_fai(FILE* f, const char* path, std::vector<FaiEntry>* out) {
  out->clear();
  std::vector<char> buf(1 << 16);
  std::string line;
  int64_t off = 0;
  bool in_seq = false, short_line = false;
  auto finish_line = [&](int64_t line_start, int64_t bytes) -> int {
    // `line` holds the line without its newline, `bytes` counts it with the newline
    if (!line.empty() && line[0] == '>') {
      FaiEntry e;
      size_t k = 1;
      while (k < line.size() && !isspace((unsigned char)line[k])) ++k;
      e.name = line.substr(1, k - 1);
      e.off = line_start + bytes;
      out->push_back(e);
      in_seq = true;
      short_line = false;
      return DCB_OK;
    }
    if (!in_seq) return line.empty() ? DCB_OK : pfail(DCB_ERR_INVALID, "%s: not a FASTA file", path);
    FaiEntry& e = out->back();
    int64_t nb = (int64_t)line.size();
    if (nb && line.back() == '\r') --nb;
    if (nb == 0) { short_line = true; return DCB_OK; }
    if (short_line) return pfail(DCB_ERR_INVALID, "%s: sequence %s has lines of different lengths", path, e.name.c_str());
    if (e.line_bases == 0) { e.line_bases = nb; e.line_width = bytes; }
    else if (nb > e.line_bases || bytes - nb != e.line_width - e.line_bases)
      return pfail(DCB_ERR_INVALID, "%s: sequence %s has lines of different lengths", path, e.name.c_str());
    if (nb < e.line_bases) short_line = true;
    e.len += nb;
    return DCB_OK;
  };
  int64_t line_start = 0;
  size_t n;
  fseeko(f, 0, SEEK_SET);
  while ((n = fread(buf.data(), 1, buf.size(), f)) > 0) {
    for (size_t i = 0; i < n; ++i) {
      if (buf[i] == '\n') {
        const int rc = finish_line(line_start, off + (int64_t)i + 1 - line_start);
        if (rc) return rc;
        line.clear();
        line_start = off + (int64_t)i + 1;
      } else {
        line.push_back(buf[i]);
      }
    }
    off += (int64_t)n;
  }
  if (!line.empty()) {
    const int rc = finish_line(line_start, off - line_start);
    if (rc) return rc;
  }
  return DCB_OK;
}

int read_fai(const std::string& path, std::vector<FaiEntry>* out) {
  FILE* f = fopen(path.c_str(), "r");
  if (!f) return 1;   // none: the caller builds the index
  char line[4096];
  int rc = DCB_OK;
  while (fgets(line, sizeof line, f)) {
    char name[4096];
    long long len, off, lb, lw;
    if (line[0] == '\n') continue;
    if (sscanf(line, "%4095s %lld %lld %lld %lld", name, &len, &off, &lb, &lw) != 5 || len < 0 || off < 0 || lb <= 0 || lw < lb) {
      rc = pfail(DCB_ERR_INVALID, "%s: malformed FASTA index line", path.c_str());
      break;
    }
    FaiEntry e;
    e.name = name; e.len = len; e.off = off; e.line_bases = lb; e.line_width = lw;
    out->push_back(e);
  }
  fclose(f);
  return rc;
}

// Bases [start, stop) of sequence e, clipped to the sequence, as the file holds them (case kept).
int fasta_fetch(dcb_calib* p, const FaiEntry& e, int64_t start, int64_t stop, std::string* out) {
  out->clear();
  start = std::max<int64_t>(start, 0);
  stop = std::min(stop, e.len);
  if (stop <= start) return DCB_OK;
  auto at = [&](int64_t k) { return e.off + k / e.line_bases * e.line_width + k % e.line_bases; };
  const int64_t b0 = at(start), b1 = at(stop - 1) + 1;
  std::string raw((size_t)(b1 - b0), '\0');
  if (fseeko(p->fa, (off_t)b0, SEEK_SET) != 0 || fread(&raw[0], 1, raw.size(), p->fa) != raw.size())
    return pfail(DCB_ERR_INVALID, "FASTA: cannot read %s:%lld-%lld", e.name.c_str(), (long long)start, (long long)stop);
  out->reserve((size_t)(stop - start));
  for (char c : raw) if (c != '\n' && c != '\r') out->push_back(c);
  if ((int64_t)out->size() != stop - start) return pfail(DCB_ERR_INVALID, "FASTA: %s does not match its index", e.name.c_str());
  return DCB_OK;
}

// The virtual offset a fetch of [lo, ...) on reference t starts reading at: the linear index's entry for lo's 16 kb
// window (or the last window's, past the end), never before the reference's first chunk.  A window with no entry
// takes the nearest earlier one, which can only start the read earlier.
uint64_t fetch_offset(const dcb_calib* p, int32_t t, int64_t lo) {
  const uint64_t first = p->first[t];
  const std::vector<uint64_t>& lin = p->linear[t];
  if (lin.empty()) return first;
  int64_t w = std::min<int64_t>(std::max<int64_t>(lo, 0) >> 14, (int64_t)lin.size() - 1);
  while (w > 0 && lin[w] == 0) --w;
  return std::max(first, lin[w]);
}

// Decode / validate the kept records [a, b) of the batch into the offsets the serial pass gave them.  Returns the index
// of the first record that fails, or -1; its message goes to *err.
int64_t export_records(dcb_calib* p, size_t a, size_t b, std::string* err) {
  for (size_t k = a; k < b; ++k) {
    const uint8_t* r = p->arena.data() + p->rec_at[k];
    int32_t* m = &p->meta[k * DCB_CALIB_META];
    const int l_name = r[8];
    p->names[k].assign(reinterpret_cast<const char*>(r + 32), l_name ? l_name - 1 : 0);
    const int32_t n_cig = m[3], l_seq = m[5];
    const uint8_t* c = r + 32 + l_name;
    memcpy(&p->cigar[m[2]], c, 4ull * n_cig);
    int64_t qlen = 0;
    for (int j = 0; j < n_cig; ++j) if (op_has_query(p->cigar[m[2] + j] & 15)) qlen += p->cigar[m[2] + j] >> 4;
    const uint8_t* s = c + 4ull * n_cig;
    const uint8_t* q = s + (l_seq + 1) / 2;
    char buf[512];
    if (l_seq == 0) snprintf(buf, sizeof buf, "read %s has no SEQ", p->names[k].c_str());
    else if (q[0] == 0xff) snprintf(buf, sizeof buf, "read %s has no QUAL", p->names[k].c_str());
    else if (qlen != l_seq)
      snprintf(buf, sizeof buf, "read %s: its cigar covers %lld query bases, its SEQ holds %d", p->names[k].c_str(),
               (long long)qlen, l_seq);
    else buf[0] = 0;
    if (buf[0]) { *err = buf; return (int64_t)k; }
    uint8_t* so = &p->seq[m[4]];
    for (int32_t i = 0; i < l_seq; ++i) so[i] = (s[i >> 1] >> (i & 1 ? 0 : 4)) & 15;
    memcpy(&p->qual[m[4]], q, (size_t)l_seq);
  }
  return -1;
}

}  // namespace

extern "C" {

int dcb_calib_open(const char* bam, const char* fasta, int32_t n_threads, dcb_calib** out) {
  if (!bam || !fasta || !out) return pfail(DCB_ERR_INVALID, "dcb_calib_open: null argument");
  if (n_threads < 1) return pfail(DCB_ERR_INVALID, "dcb_calib_open: %d threads; need at least 1", n_threads);
  dcb_calib* p = new dcb_calib();
  p->n_threads = std::min(n_threads, 256);
  int rc = p->bam.open(bam);
  if (!rc) rc = read_bai(std::string(bam) + ".bai", p->bam.refs.size(), &p->first, &p->linear);
  if (!rc && !(p->fa = fopen(fasta, "rb"))) rc = pfail(DCB_ERR_INVALID, "cannot open %s", fasta);
  if (!rc) {
    uint8_t magic[2] = {0, 0};
    if (fread(magic, 1, 2, p->fa) == 2 && magic[0] == 0x1f && magic[1] == 0x8b)
      rc = pfail(DCB_ERR_INVALID, "%s is compressed; a bgzipped FASTA is not supported, decompress it", fasta);
  }
  if (!rc) {
    const int fr = read_fai(std::string(fasta) + ".fai", &p->fai);
    if (fr == 1) rc = build_fai(p->fa, fasta, &p->fai);
    else rc = fr;
  }
  if (rc) { delete p; return rc; }
  for (size_t t = 0; t < p->bam.refs.size(); ++t) {
    p->tid[p->bam.refs[t]] = (int32_t)t;
    p->bam_contigs += p->bam.refs[t] + "\t" + std::to_string(p->bam.ref_len[t]) + "\n";
  }
  for (const FaiEntry& e : p->fai) p->fasta_contigs += e.name + "\t" + std::to_string(e.len) + "\n";
  *out = p;
  return DCB_OK;
}

void dcb_calib_close(dcb_calib* p) { delete p; }

const char* dcb_calib_contigs(dcb_calib* p, int32_t fasta) {
  if (!p) return "";
  return fasta ? p->fasta_contigs.c_str() : p->bam_contigs.c_str();
}

int dcb_calib_fetch_reference(dcb_calib* p, const char* contig, int64_t start, int64_t stop, uint8_t* out, int64_t* n) {
  if (!p || !contig || !n || stop < start) return pfail(DCB_ERR_INVALID, "dcb_calib_fetch_reference: bad argument");
  *n = 0;
  for (const FaiEntry& e : p->fai) {
    if (e.name != contig) continue;
    std::string s;
    const int rc = fasta_fetch(p, e, start, stop, &s);
    if (rc) return rc;
    if (out && !s.empty()) memcpy(out, s.data(), s.size());
    *n = (int64_t)s.size();
    return DCB_OK;
  }
  return pfail(DCB_ERR_INVALID, "contig %s is not in the FASTA file", contig);
}

int dcb_calib_query(dcb_calib* p, const char* contig, int64_t start, int64_t stop, int64_t min_pos, int32_t min_mapq) {
  if (!p || !contig || stop < start) return pfail(DCB_ERR_INVALID, "dcb_calib_query: bad argument");
  auto it = p->tid.find(contig);
  if (it == p->tid.end()) return pfail(DCB_ERR_INVALID, "contig %s is not in the BAM header", contig);
  p->q_tid = it->second;
  p->q_lo = start; p->q_hi = stop; p->q_min_pos = min_pos; p->q_min_mapq = min_mapq;
  p->q_done = stop == start || p->first[p->q_tid] == UINT64_MAX;
  if (!p->q_done && !p->bam.z.seek(fetch_offset(p, p->q_tid, start)))
    return pfail(DCB_ERR_INVALID, "BAM: bad index offset for %s", contig);
  return DCB_OK;
}

int dcb_calib_next_batch(dcb_calib* p, int64_t max_bases, int64_t* sizes) {
  if (!p || !sizes || max_bases < 1) return pfail(DCB_ERR_INVALID, "dcb_calib_next_batch: bad argument");
  sizes[0] = sizes[1] = sizes[2] = 0;
  p->arena.clear(); p->rec_at.clear(); p->meta.clear();
  max_bases = std::min<int64_t>(max_bases, 1 << 30);
  int64_t n_cig = 0, n_bases = 0;
  // Serial pass: inflate, select, and give every kept record its place in the flat arrays.
  while (!p->q_done && n_bases < max_bases) {
    const size_t at = p->arena.size();
    const int rc = p->bam.next_raw(&p->arena);
    if (rc < 0) return rc;
    if (rc == 0) { p->q_done = true; break; }
    const uint8_t* r = p->arena.data() + at;
    int32_t refid, pos, l_seq;
    uint16_t flag, nc;
    memcpy(&refid, r, 4); memcpy(&pos, r + 4, 4); memcpy(&nc, r + 12, 2); memcpy(&flag, r + 14, 2); memcpy(&l_seq, r + 16, 4);
    const int mapq = r[9];
    if (refid != p->q_tid || pos >= p->q_hi) {
      p->arena.resize(at);
      if (refid < 0 || refid > p->q_tid || (refid == p->q_tid && pos >= p->q_hi)) p->q_done = true;
      continue;
    }
    // AlignmentFile.fetch(contig, lo, hi) returns a record when htslib's overlap test holds: pos < hi and
    // endpos > lo, where endpos (bam_endpos) is pos plus the cigar's reference length, or pos + 1 when that is 0 or
    // the record is unmapped.
    const int64_t rlen = (flag & 4) ? 0 : raw_ref_len(r);
    const int64_t endpos = pos + (rlen ? rlen : 1);
    if (endpos <= p->q_lo || pos < p->q_min_pos || (flag & kCalibSkipFlags) || mapq < p->q_min_mapq) {
      p->arena.resize(at);
      continue;
    }
    if (endpos > INT32_MAX) return pfail(DCB_ERR_INVALID, "a record at %d reaches past 2^31", pos);
    p->rec_at.push_back(at);
    const int32_t m[DCB_CALIB_META] = {pos, (int32_t)endpos, (int32_t)n_cig, nc, (int32_t)n_bases, l_seq};
    p->meta.insert(p->meta.end(), m, m + DCB_CALIB_META);
    n_cig += nc;
    n_bases += l_seq;
  }
  const size_t n = p->rec_at.size();
  p->cigar.resize((size_t)n_cig); p->seq.resize((size_t)n_bases); p->qual.resize((size_t)n_bases);
  p->names.assign(n, std::string());
  // Parallel pass: decode and validate on n_threads threads, contiguous slices of the batch; the first failing record
  // in batch order is reported, whichever thread found it.
  const int nt = (int)std::min<size_t>((size_t)p->n_threads, std::max<size_t>(n, 1));
  std::vector<int64_t> bad(nt, -1);
  std::vector<std::string> errs(nt);
  auto work = [&](int t) { bad[t] = export_records(p, n * t / nt, n * (t + 1) / nt, &errs[t]); };
  if (nt == 1) {
    work(0);
  } else {
    std::vector<std::thread> th;
    for (int t = 0; t < nt; ++t) th.emplace_back(work, t);
    for (auto& x : th) x.join();
  }
  for (int t = 0; t < nt; ++t) if (bad[t] >= 0) return pfail(DCB_ERR_INVALID, "%s", errs[t].c_str());
  sizes[0] = (int64_t)n; sizes[1] = n_cig; sizes[2] = n_bases;
  return n ? 1 : 0;
}

int dcb_calib_get_batch(dcb_calib* p, int32_t* read_meta, uint32_t* cigar, uint8_t* seq, uint8_t* qual) {
  if (!p) return pfail(DCB_ERR_INVALID, "dcb_calib_get_batch: null handle");
  if (read_meta && !p->meta.empty()) memcpy(read_meta, p->meta.data(), p->meta.size() * sizeof(int32_t));
  if (cigar && !p->cigar.empty()) memcpy(cigar, p->cigar.data(), p->cigar.size() * sizeof(uint32_t));
  if (seq && !p->seq.empty()) memcpy(seq, p->seq.data(), p->seq.size());
  if (qual && !p->qual.empty()) memcpy(qual, p->qual.data(), p->qual.size());
  return DCB_OK;
}

const char* dcb_calib_read_name(dcb_calib* p, int64_t i) {
  if (!p || i < 0 || i >= (int64_t)p->names.size()) return "";
  return p->names[(size_t)i].c_str();
}

}  // extern "C"

// ----------------------------------------------------------------------------------------------- sequence reader
// The host side of `kmer_qv` (include/dcb200.h "k-mer QV"): the reads of one FASTA, FASTQ or BAM file, in file order,
// exported in batches of concatenated bases, Phred qualities and offsets.  The format comes from the content: a BGZF
// stream that inflates to "BAM\1" is a BAM, anything else is read through zlib's gz* reader (plain or gzip text), where
// '>' starts a FASTA file and '@' a FASTQ file.
struct dcb_seq_reader {
  std::string path;
  bool bam_mode = false, fastq = false, done = false;
  BamReader bam;
  gzFile gz = nullptr;
  std::vector<char> buf;
  size_t at = 0, got = 0;
  bool eof = false;
  std::string pending;              // FASTA: the header line that starts the next record
  int64_t line_no = 0;
  // the current batch
  std::vector<uint8_t> seq, qual, has_qual;
  std::vector<int64_t> off;
  std::vector<std::string> names;
  ~dcb_seq_reader() { if (gz) gzclose(gz); }

  // One line without its newline (and '\r'): 1 = line, 0 = end of the file, < 0 = error.  A gzip stream that is
  // corrupt (a bad CRC or bad data) or ends before its end is an error, never a shorter file.
  int getline(std::string* line) {
    line->clear();
    bool any = false;
    for (;;) {
      if (at == got) {
        if (eof) break;
        const int n = gzread(gz, buf.data(), (unsigned)buf.size());
        if (n <= 0) {
          int err = Z_OK;
          const char* msg = gzerror(gz, &err);
          if (n < 0 || err != Z_OK)
            return pfail(DCB_ERR_INVALID, "%s: cannot read past line %lld: %s", path.c_str(), (long long)line_no,
                         msg && *msg ? msg : "read error");
          eof = true;
          break;
        }
        at = 0; got = (size_t)n;
      }
      any = true;
      const char* s = buf.data() + at;
      const char* nl = static_cast<const char*>(memchr(s, '\n', got - at));
      if (nl) { line->append(s, nl - s); at += (nl - s) + 1; break; }
      line->append(s, got - at);
      at = got;
    }
    if (!any) return 0;
    ++line_no;
    if (!line->empty() && line->back() == '\r') line->pop_back();
    return 1;
  }
};

namespace {

std::string header_name(const std::string& line) {
  size_t k = 1;
  while (k < line.size() && !isspace((unsigned char)line[k])) ++k;
  return line.substr(1, k - 1);
}

void append_bases(dcb_seq_reader* p, const char* s, size_t n) {
  for (size_t i = 0; i < n; ++i) p->seq.push_back((uint8_t)toupper((unsigned char)s[i]));
}

// The next record of a text file into the batch: 1 = record, 0 = end of file, < 0 = error.
int next_text_record(dcb_seq_reader* p) {
  std::string line;
  int rc;
  if (p->fastq) {
    do { if ((rc = p->getline(&line)) <= 0) return rc; } while (line.empty());
    if (line[0] != '@') return pfail(DCB_ERR_INVALID, "%s:%lld: a FASTQ record must start with '@'", p->path.c_str(), (long long)p->line_no);
    const std::string name = header_name(line);
    std::string s, plus, q;
    for (std::string* l : {&s, &plus, &q}) {
      if ((rc = p->getline(l)) < 0) return rc;
      if (rc == 0 || (l == &plus && (plus.empty() || plus[0] != '+')))
        return pfail(DCB_ERR_INVALID, "%s: FASTQ record %s is truncated", p->path.c_str(), name.c_str());
    }
    if (q.size() != s.size())
      return pfail(DCB_ERR_INVALID, "%s: FASTQ record %s has %zu bases and %zu qualities", p->path.c_str(), name.c_str(),
                   s.size(), q.size());
    append_bases(p, s.data(), s.size());
    for (char c : q) {
      if ((unsigned char)c < 33 || (unsigned char)c > 126)
        return pfail(DCB_ERR_INVALID, "%s: FASTQ record %s has a quality character outside '!'..'~'", p->path.c_str(), name.c_str());
      p->qual.push_back((uint8_t)(c - 33));
    }
    p->names.push_back(name);
    p->has_qual.push_back(1);
    return 1;
  }
  if (p->pending.empty()) {
    do { if ((rc = p->getline(&line)) <= 0) return rc; } while (line.empty());
    if (line[0] != '>') return pfail(DCB_ERR_INVALID, "%s:%lld: a FASTA record must start with '>'", p->path.c_str(), (long long)p->line_no);
    p->pending = line;
  }
  p->names.push_back(header_name(p->pending));
  p->pending.clear();
  while ((rc = p->getline(&line)) > 0) {
    if (!line.empty() && line[0] == '>') { p->pending = line; break; }
    append_bases(p, line.data(), line.size());
  }
  if (rc < 0) return rc;
  p->qual.resize(p->seq.size(), 0);
  p->has_qual.push_back(0);
  return 1;
}

// The next record of a BAM file into the batch: secondary and supplementary records are skipped.
int next_bam_record(dcb_seq_reader* p) {
  BamRecord r;
  for (;;) {
    const int rc = p->bam.next(&r);
    if (rc < 0) return pfail(DCB_ERR_INVALID, "%s: %s", p->path.c_str(), g_prep_error.c_str());
    if (rc == 0) return 0;
    if (!(r.flag & (0x100 | 0x800))) break;
  }
  if (r.seq.empty()) return pfail(DCB_ERR_INVALID, "%s: read %s has no SEQ", p->path.c_str(), r.qname.c_str());
  append_bases(p, r.seq.data(), r.seq.size());
  const bool q = r.qual[0] != 0xff;
  if (q) p->qual.insert(p->qual.end(), r.qual.begin(), r.qual.end());
  else p->qual.resize(p->seq.size(), 0);
  p->names.push_back(r.qname);
  p->has_qual.push_back(q ? 1 : 0);
  return 1;
}

}  // namespace

extern "C" {

int dcb_seq_open(const char* path, dcb_seq_reader** out) {
  if (!path || !out) return pfail(DCB_ERR_INVALID, "dcb_seq_open: null argument");
  *out = nullptr;
  std::unique_ptr<dcb_seq_reader> p(new dcb_seq_reader());
  p->path = path;
  FILE* f = fopen(path, "rb");
  if (!f) return pfail(DCB_ERR_INVALID, "cannot open %s", path);
  uint8_t magic[4] = {0, 0, 0, 0};
  const size_t n = fread(magic, 1, 4, f);
  fclose(f);
  if (n == 4 && magic[0] == 31 && magic[1] == 139 && (magic[3] & 4)) {   // BGZF: BAM or a bgzipped text file
    gzFile g = gzopen(path, "rb");
    char head[4] = {0, 0, 0, 0};
    const bool is_bam = g && gzread(g, head, 4) == 4 && memcmp(head, "BAM\1", 4) == 0;
    if (g) gzclose(g);
    if (is_bam) {
      p->bam_mode = true;
      const int rc = p->bam.open(path);
      if (rc) return rc;
      *out = p.release();
      return DCB_OK;
    }
  }
  if (!(p->gz = gzopen(path, "rb"))) return pfail(DCB_ERR_INVALID, "cannot open %s", path);
  p->buf.resize(1 << 20);
  std::string line;
  int rc;
  while ((rc = p->getline(&line)) > 0 && line.empty()) {}
  if (rc < 0) return rc;
  if (line.empty()) { p->done = true; *out = p.release(); return DCB_OK; }   // an empty file holds no reads
  if (line[0] == '@') {
    p->fastq = true;
    gzrewind(p->gz);
    p->at = p->got = 0; p->eof = false; p->line_no = 0;
  } else if (line[0] == '>') {
    p->pending = line;
  } else {
    return pfail(DCB_ERR_INVALID, "%s is not a FASTA, FASTQ or BAM file", path);
  }
  *out = p.release();
  return DCB_OK;
}

int dcb_seq_next_batch(dcb_seq_reader* p, int64_t max_bases, int64_t* sizes) {
  if (!p || !sizes || max_bases < 1) return pfail(DCB_ERR_INVALID, "dcb_seq_next_batch: bad argument");
  sizes[0] = sizes[1] = 0;
  p->seq.clear(); p->qual.clear(); p->has_qual.clear(); p->names.clear();
  p->off.assign(1, 0);
  max_bases = std::min<int64_t>(max_bases, (int64_t)1 << 31);
  while (!p->done && (int64_t)p->seq.size() < max_bases) {
    const int rc = p->bam_mode ? next_bam_record(p) : next_text_record(p);
    if (rc < 0) return rc;
    if (rc == 0) { p->done = true; break; }
    p->off.push_back((int64_t)p->seq.size());
  }
  sizes[0] = (int64_t)p->names.size();
  sizes[1] = (int64_t)p->seq.size();
  return sizes[0] ? 1 : 0;
}

int dcb_seq_get_batch(dcb_seq_reader* p, uint8_t* bases, uint8_t* qual, int64_t* offsets, uint8_t* has_qual) {
  if (!p) return pfail(DCB_ERR_INVALID, "dcb_seq_get_batch: null handle");
  if (bases && !p->seq.empty()) memcpy(bases, p->seq.data(), p->seq.size());
  if (qual && !p->qual.empty()) memcpy(qual, p->qual.data(), p->qual.size());
  if (offsets) memcpy(offsets, p->off.data(), p->off.size() * sizeof(int64_t));
  if (has_qual && !p->has_qual.empty()) memcpy(has_qual, p->has_qual.data(), p->has_qual.size());
  return DCB_OK;
}

const char* dcb_seq_read_name(dcb_seq_reader* p, int64_t i) {
  if (!p || i < 0 || i >= (int64_t)p->names.size()) return "";
  return p->names[(size_t)i].c_str();
}

void dcb_seq_close(dcb_seq_reader* p) { delete p; }

}  // extern "C"
