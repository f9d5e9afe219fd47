// bam.cu -- `checkm coverage` (checkm/coverage.py:57-287) and `checkm gc_bias_plot`'s read depth per window: BGZF blocks
// inflated on the device, BAM records walked and classified on the device, nine integer counters per reference.
//
// Layout.  The caller hands over one batch: the compressed bytes of consecutive BGZF blocks, their table (file offset,
// length, ISIZE; ckm_bgzf_blocks) and the record segments to walk.  Block b inflates to out[U[b] .. U[b] + ISIZE[b]),
// U the exclusive prefix sum of ISIZE over the batch, so the batch becomes one contiguous slice of the BAM's
// decompressed stream.
//
// Kernels.
//   bgzf_inflate_kernel  one BGZF block per warp.  Lane 0 decodes the deflate stream (stored, fixed and dynamic blocks)
//                        with canonical (count, symbol) tables in shared memory; it writes literals straight to the
//                        output and queues matches, which the whole warp then copies in order (out[p + i] =
//                        out[p - d + i % d], so an overlapping match reads only bytes already written).  The warp builds
//                        each table together: per-length counts with __match_any_sync, a shuffle scan for the first
//                        slots, then a ranked placement.  Every read of compressed bits stays inside the block's
//                        payload (bits past its end read as zero and fail the final check) and every write is checked
//                        against ISIZE; a malformed block sets its status and the first bad block's index.  Last, each
//                        lane takes the CRC32 of one slice of the output and lane 0 joins the 32 partial CRCs with the
//                        shift operators x^(8n) mod P (zlib's crc32_combine), compared with the block's CRC field.
//   The record walk      one thread per segment [anchor_i, anchor_i+1) (`walk`, shared by the two kernels below): walks the
//                        records, validates each, hands it to the kernel's rule to classify, and keeps the counters in
//                        registers while refID stays the same; they go out with 64-bit atomics when it changes.  A walk
//                        must land exactly on the segment's end.  The first segment starts at the end of the header, so
//                        by induction every anchor (a record start taken from the BAI's linear index) and every record
//                        start is verified; an index that belongs to another file, or a truncated file, gives
//                        CKM_EFORMAT, never a wrong table.  The walk stops at the first record with refID -1 (the
//                        unplaced tail).
//   bam_scan_kernel      the walk with coverage.py:206-230's classification (CoverageRule).
//   bam_window_kernel    the walk with `checkm gc_bias_plot`'s read depth (coverageWindows.py:55-79, WindowRule):
//                        coverageWindows' classification and the fetch rule of `fetch(ref, 0, len)`.  Each mapped read
//                        adds its clipped span [pos, min(pos + alen, len)) to its reference's covered bases and each
//                        window's overlap with it to an int64 window array.  The thread keeps one (window, partial sum) in
//                        registers and flushes it with a 64-bit atomic when the window changes; the reads are
//                        coordinate-sorted, so most reads land in the cached window.  Walkers of neighbouring segments
//                        may share a window (segments end on 16 kbp index windows, not on W), and the atomics make that
//                        correct.
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>
#include "engine.hpp"
#include "pool.hpp"

using namespace ckm;

namespace {

constexpr int IW = 8;                         // warps (BGZF blocks) per inflate CTA
constexpr int QN = 64;                        // matches queued by lane 0 before the warp copies them
constexpr int SCAN_THREADS = 128;
constexpr int NCNT = 9;                       // reads, duplicates, secondary, failed QC, failed alignment length,
                                              // failed edit distance, failed proper pair, mapped, aligned bases
constexpr uint32_t CRC_POLY = 0xEDB88320u;

__constant__ uint16_t LBASE[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99,
                                   115, 131, 163, 195, 227, 258};
__constant__ uint8_t LEXT[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint16_t DBASE[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537,
                                   2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
__constant__ uint8_t DEXT[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12,
                                 13, 13};
__constant__ uint8_t CLORDER[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

// per-block status codes (the host turns them into messages)
enum { IF_OK = 0, IF_HEADER, IF_STORED_LEN, IF_STORED_OVER, IF_BTYPE, IF_COUNTS, IF_CLCODE, IF_LENS, IF_REPEAT,
       IF_NO_EOB, IF_LITCODE, IF_DISTCODE, IF_SYMBOL, IF_DIST_BACK, IF_OUT_OVER, IF_IN_OVER, IF_ISIZE, IF_CRC, IF_NCODES };

const char *inflate_msg(int c) {
  static const char *m[IF_NCODES] = {"ok", "bad BGZF header", "stored block length check fails", "stored block runs past the block",
                                     "reserved deflate block type", "too many length or distance codes",
                                     "bad code-length code", "bad code lengths", "length repeat with no previous length",
                                     "no end-of-block code", "bad literal/length code", "bad distance code",
                                     "invalid symbol", "distance reaches before the block", "output exceeds ISIZE",
                                     "compressed data runs past the block", "output is shorter than ISIZE", "CRC32 mismatch"};
  return c >= 0 && c < IF_NCODES ? m[c] : "unknown";
}

struct alignas(8) Match { uint32_t pos; uint16_t len; uint16_t dist; };

struct WarpTables {
  uint8_t lens[320];                          // literal/length code lengths, then distance code lengths
  uint8_t cl[20];                             // code-length code lengths
  uint16_t lcount[16], dcount[16], offs[16];
  uint16_t lsym[288], dsym[32];
  Match q[QN];
};

struct InflateParams {
  const uint8_t *comp; int64_t comp_base;     // comp[0] is the byte at file offset comp_base
  const ckm_bgzf_block *blocks; const int64_t *uoff; int64_t nblocks;
  uint8_t *out;
  int *status;                                // per block
  unsigned long long *first_bad;              // smallest index of a bad block
  uint32_t x2n[32];                           // x^(2^k) mod P
};

// bit reader of lane 0: bits past the payload read as zero; the caller checks the consumed count at the end
struct BitIn {
  const uint8_t *src; int n; int ip; int cnt; uint64_t buf;
  __device__ __forceinline__ void need(int k) {
    while (cnt < k) { const uint64_t b = ip < n ? src[ip] : 0u; ++ip; buf |= b << cnt; cnt += 8; }
  }
  __device__ __forceinline__ uint32_t bits(int k) { need(k); const uint32_t v = (uint32_t)(buf & ((1ull << k) - 1)); buf >>= k; cnt -= k; return v; }
  // canonical decode, one bit at a time (codes are stored MSB first)
  __device__ __forceinline__ int decode(const uint16_t *count, const uint16_t *sym) {
    need(15);
    int code = 0, first = 0, index = 0;
    uint64_t b = buf;
#pragma unroll 1
    for (int len = 1; len <= 15; ++len) {
      code |= (int)(b & 1); b >>= 1;
      const int c = count[len];
      if (code - c < first) { buf >>= len; cnt -= len; return sym[index + (code - first)]; }
      index += c; first += c; first <<= 1; code <<= 1;
    }
    return -1;
  }
};

// Warp-collective canonical table: count[len], sym[] in (length, symbol) order.  Returns (all lanes) the number of unused
// codes: 0 complete, > 0 incomplete, < 0 over-subscribed.  *nonzero: symbols with a code; *ones: codes of length 1.
__device__ int warp_build(const uint8_t *lens, int n, uint16_t *count, uint16_t *sym, uint16_t *offs, int lane, int *ones,
                          int *nonzero) {
  if (lane < 16) count[lane] = 0;
  __syncwarp();
  for (int base = 0; base < n; base += 32) {
    const int s = base + lane;
    const int L = s < n ? lens[s] : 0;
    const unsigned m = __match_any_sync(0xFFFFFFFFu, L);
    if (L && lane == __ffs(m) - 1) count[L] += (uint16_t)__popc(m);
    __syncwarp();
  }
  const int c = (lane >= 1 && lane < 16) ? count[lane] : 0;
  int scan = c;                                           // inclusive scan over lanes 1..15
#pragma unroll
  for (int o = 1; o < 16; o <<= 1) { const int v = __shfl_up_sync(0xFFFFFFFFu, scan, o); if (lane >= o) scan += v; }
  if (lane < 16) offs[lane] = (uint16_t)(scan - c);      // first slot of length `lane`
  int left = 1;
  for (int len = 1; len < 16; ++len) {
    left <<= 1; left -= __shfl_sync(0xFFFFFFFFu, c, len);
    if (left < 0) break;
  }
  *ones = __shfl_sync(0xFFFFFFFFu, c, 1);
  *nonzero = __shfl_sync(0xFFFFFFFFu, scan, 15);
  __syncwarp();
  if (left < 0) return left;
  const unsigned lt = (1u << lane) - 1u;
  for (int base = 0; base < n; base += 32) {
    const int s = base + lane;
    const int L = s < n ? lens[s] : 0;
    const unsigned m = __match_any_sync(0xFFFFFFFFu, L);
    if (L) sym[offs[L] + __popc(m & lt)] = (uint16_t)s;
    __syncwarp();
    if (L && lane == __ffs(m) - 1) offs[L] += (uint16_t)__popc(m);
    __syncwarp();
  }
  return left;
}

__device__ __forceinline__ uint32_t multmodp(uint32_t a, uint32_t b) {
  uint32_t m = 1u << 31, p = 0;
  for (;;) {
    if (a & m) { p ^= b; if ((a & (m - 1)) == 0) break; }
    m >>= 1;
    b = b & 1 ? (b >> 1) ^ CRC_POLY : b >> 1;
  }
  return p;
}

__global__ void __launch_bounds__(IW * 32) bgzf_inflate_kernel(InflateParams p) {
  __shared__ uint32_t crc_tab[256];
  __shared__ WarpTables wt_all[IW];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) {
    uint32_t c = (uint32_t)i;
    for (int k = 0; k < 8; ++k) c = c & 1 ? (c >> 1) ^ CRC_POLY : c >> 1;
    crc_tab[i] = c;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int64_t b = (int64_t)blockIdx.x * IW + (threadIdx.x >> 5);
  if (b >= p.nblocks) return;
  WarpTables &w = wt_all[threadIdx.x >> 5];
  const ckm_bgzf_block blk = p.blocks[b];
  const uint8_t *bp = p.comp + (blk.coffset - p.comp_base);        // the host checked that the block lies in comp
  const int clen = blk.clen, isize = blk.isize;
  uint8_t *out = p.out + p.uoff[b];
  const int xlen = bp[10] | bp[11] << 8;
  int err = (12 + xlen + 8 > clen) ? IF_HEADER : IF_OK;
  BitIn in;
  in.src = bp + 12 + xlen; in.n = clen - 20 - xlen; in.ip = 0; in.cnt = 0; in.buf = 0;
  int op = 0;                                                      // output position (lane 0's copy is authoritative)
  bool last = false;
  while (!err && !last) {
    int btype = 0;
    if (lane == 0) { last = in.bits(1); btype = (int)in.bits(2); }
    last = __shfl_sync(0xFFFFFFFFu, last, 0);
    btype = __shfl_sync(0xFFFFFFFFu, btype, 0);
    if (btype == 0) {                                              // stored
      int len = 0, sp = 0;
      if (lane == 0) {
        in.buf >>= (in.cnt & 7); in.cnt &= ~7;
        const uint32_t ln = in.bits(16), nl = in.bits(16);
        in.ip -= in.cnt >> 3; in.buf = 0; in.cnt = 0;              // give back whole bytes read ahead
        len = (int)ln; sp = in.ip;
        if (ln != (~nl & 0xFFFFu)) err = IF_STORED_LEN;
        else if (sp + len > in.n) err = IF_STORED_OVER;
        else if (op + len > isize) err = IF_OUT_OVER;
      }
      err = __shfl_sync(0xFFFFFFFFu, err, 0);
      len = __shfl_sync(0xFFFFFFFFu, len, 0); sp = __shfl_sync(0xFFFFFFFFu, sp, 0);
      const int o = __shfl_sync(0xFFFFFFFFu, op, 0);
      if (err) break;
      for (int i = lane; i < len; i += 32) out[o + i] = in.src[sp + i];
      if (lane == 0) { in.ip += len; op += len; }
      __syncwarp();
      continue;
    }
    if (btype == 3) { err = IF_BTYPE; break; }
    int nlen = 288, ndist = 30;
    if (btype == 1) {
      for (int i = lane; i < 318; i += 32) w.lens[i] = i < 144 ? 8 : i < 256 ? 9 : i < 280 ? 7 : i < 288 ? 8 : 5;
      __syncwarp();
    } else {
      int hclen = 0;
      if (lane == 0) {
        nlen = (int)in.bits(5) + 257; ndist = (int)in.bits(5) + 1; hclen = (int)in.bits(4) + 4;
        if (nlen > 286 || ndist > 30) err = IF_COUNTS;
        else for (int i = 0; i < 19; ++i) w.cl[CLORDER[i]] = i < hclen ? (uint8_t)in.bits(3) : 0;
      }
      err = __shfl_sync(0xFFFFFFFFu, err, 0);
      nlen = __shfl_sync(0xFFFFFFFFu, nlen, 0); ndist = __shfl_sync(0xFFFFFFFFu, ndist, 0);
      if (err) break;
      __syncwarp();
      int ones, nz;
      if (warp_build(w.cl, 19, w.dcount, w.dsym, w.offs, lane, &ones, &nz) != 0) { err = IF_CLCODE; break; }
      if (lane == 0) {
        int i = 0;
        while (i < nlen + ndist) {
          const int sym = in.decode(w.dcount, w.dsym);
          if (sym < 0) { err = IF_LENS; break; }
          if (sym < 16) { w.lens[i++] = (uint8_t)sym; continue; }
          int l = 0, rep;
          if (sym == 16) { if (i == 0) { err = IF_REPEAT; break; } l = w.lens[i - 1]; rep = 3 + (int)in.bits(2); }
          else if (sym == 17) rep = 3 + (int)in.bits(3);
          else rep = 11 + (int)in.bits(7);
          if (i + rep > nlen + ndist) { err = IF_LENS; break; }
          while (rep--) w.lens[i++] = (uint8_t)l;
        }
        if (!err && w.lens[256] == 0) err = IF_NO_EOB;
        if (!err && in.ip > in.n + 8) err = IF_IN_OVER;
      }
      err = __shfl_sync(0xFFFFFFFFu, err, 0);
      if (err) break;
      __syncwarp();
    }
    {
      int ones, nz;
      const int left = warp_build(w.lens, nlen, w.lcount, w.lsym, w.offs, lane, &ones, &nz);
      if (left < 0 || (btype == 2 && left > 0 && nz != ones)) { err = IF_LITCODE; break; }
      const int dleft = warp_build(w.lens + nlen, ndist, w.dcount, w.dsym, w.offs, lane, &ones, &nz);
      if (dleft < 0 || (btype == 2 && dleft > 0 && nz != ones)) { err = IF_DISTCODE; break; }
    }
    bool done = false;
    while (!done) {
      int nq = 0;
      if (lane == 0) {
        while (nq < QN) {
          int sym = in.decode(w.lcount, w.lsym);
          if (sym < 0) { err = IF_LITCODE; break; }
          if (sym < 256) {
            if (op >= isize) { err = IF_OUT_OVER; break; }
            out[op++] = (uint8_t)sym;
            continue;
          }
          if (sym == 256) { done = true; break; }
          sym -= 257;
          if (sym >= 29) { err = IF_SYMBOL; break; }
          const int len = LBASE[sym] + (int)in.bits(LEXT[sym]);
          const int ds = in.decode(w.dcount, w.dsym);
          if (ds < 0) { err = IF_DISTCODE; break; }
          if (ds >= 30) { err = IF_SYMBOL; break; }
          const int dist = DBASE[ds] + (int)in.bits(DEXT[ds]);
          if (dist > op) { err = IF_DIST_BACK; break; }
          if (op + len > isize) { err = IF_OUT_OVER; break; }
          w.q[nq].pos = (uint32_t)op; w.q[nq].len = (uint16_t)len; w.q[nq].dist = (uint16_t)dist; ++nq;
          op += len;
          if (in.ip > in.n + 8) { err = IF_IN_OVER; break; }
        }
      }
      nq = __shfl_sync(0xFFFFFFFFu, nq, 0);
      done = __shfl_sync(0xFFFFFFFFu, done, 0);
      err = __shfl_sync(0xFFFFFFFFu, err, 0);
      __syncwarp();
      for (int j = 0; j < nq; ++j) {                               // queued matches are valid even when a later token is not
        const Match m = w.q[j];
        const int d = m.dist, L = m.len;
        uint8_t *dst = out + m.pos;
        const uint8_t *src = dst - d;
        for (int i = lane; i < L; i += 32) dst[i] = src[d >= L ? i : i % d];
        __syncwarp();
      }
      if (err) break;
    }
  }
  if (!err && lane == 0) {
    if ((int64_t)in.ip * 8 - in.cnt > (int64_t)in.n * 8) err = IF_IN_OVER;
    else if (op != isize) err = IF_ISIZE;
  }
  err = __shfl_sync(0xFFFFFFFFu, err, 0);
  if (!err) {
    const uint8_t *t = bp + clen - 8;
    const uint32_t want = (uint32_t)t[0] | (uint32_t)t[1] << 8 | (uint32_t)t[2] << 16 | (uint32_t)t[3] << 24;
    const uint32_t isz = (uint32_t)t[4] | (uint32_t)t[5] << 8 | (uint32_t)t[6] << 16 | (uint32_t)t[7] << 24;
    const int S = (isize + 31) / 32;
    const int a = min(isize, lane * S), e = min(isize, a + S);
    uint32_t c = 0xFFFFFFFFu;
    for (int i = a; i < e; ++i) c = crc_tab[(c ^ out[i]) & 0xFF] ^ (c >> 8);
    c ^= 0xFFFFFFFFu;
    // x^(8 * len) mod P for this lane's slice length: zlib's x2nmodp(len, 3)
    uint32_t op8 = 1u << 31;
    for (int n = e - a, k = 3; n; n >>= 1, ++k)
      if (n & 1) op8 = multmodp(p.x2n[k & 31], op8);
    uint32_t crc = 0;
    for (int l = 0; l < 32; ++l) {                                 // crc(AB) = x^(8|B|) crc(A) ^ crc(B)
      const uint32_t cl = __shfl_sync(0xFFFFFFFFu, c, l), ol = __shfl_sync(0xFFFFFFFFu, op8, l);
      if (lane == 0) crc = l == 0 ? cl : multmodp(ol, crc) ^ cl;
    }
    if (lane == 0 && (crc != want || isz != (uint32_t)isize)) err = IF_CRC;
    err = __shfl_sync(0xFFFFFFFFu, err, 0);
  }
  if (lane == 0) {
    p.status[b] = err;
    if (err) atomicMin(p.first_bad, (unsigned long long)b);
  }
}

// ---- the record walk ----
enum { SC_TAIL = -1, SC_OK = 0, SC_RECORD, SC_REFID, SC_UNPLACED, SC_NO_NM, SC_ANCHOR, SC_AUX, SC_NO_NUM_NM, SC_NO_CIGAR,
       SC_NEG_POS, SC_NCODES };

const char *scan_msg(int c) {
  static const char *m[SC_NCODES] = {"ok", "malformed BAM record", "refID out of range",
                                     "unplaced read before the end of the placed reads", "no integer NM tag",
                                     "the record walk does not land on the next index anchor (index of another file?)",
                                     "malformed auxiliary field", "no numeric NM tag (types c, C, s, S, i, I or f)",
                                     "no CIGAR, so no alignment length", "mapped read at a negative position"};
  return c >= 0 && c < SC_NCODES ? m[c] : "unknown";
}

// codes whose message names the read
bool scan_names_read(int c) { return c == SC_NO_NM || c == SC_NO_NUM_NM || c == SC_NO_CIGAR || c == SC_NEG_POS; }

// the parameters of both walk kernels
struct WalkParams {
  const uint8_t *data;                        // 4-byte aligned, readable 8 bytes past the last segment end
  const int64_t *seg_start, *seg_end; int64_t nseg;
  int32_t n_ref; ckm_bam_filter filter;
  unsigned long long *counters;               // n_ref x NCNT
  unsigned long long *err;                    // min of (record position << 8 | code)
};

__device__ __forceinline__ uint32_t ld32(const uint8_t *d, int64_t p) {
  const int64_t a = p & ~3ll;
  const uint32_t w0 = *reinterpret_cast<const uint32_t *>(d + a), w1 = *reinterpret_cast<const uint32_t *>(d + a + 4);
  return __funnelshift_r(w0, w1, (uint32_t)(p & 3) * 8);
}

// query_alignment_length: pysam's query end minus query start.  Leading soft clips (hard clips skipped) give the start;
// l_seq minus the trailing soft clips (down to the second op) gives the end.  Without SEQ (l_seq == 0) the query length is
// taken from the CIGAR: the M, I, =, X ops, i.e. the length SEQ would have without its soft clips (DESIGN §9).
__device__ __forceinline__ int64_t aligned_length(const uint8_t *d, int64_t cig, int nc, int32_t l_seq) {
  if (l_seq == 0) {
    int64_t s = 0;
    for (int k = 0; k < nc; ++k) {
      const uint32_t c = ld32(d, cig + 4ll * k), o = c & 15u;
      if (o == 0 || o == 1 || o == 7 || o == 8) s += c >> 4;
    }
    return s;
  }
  int64_t start = 0, end = l_seq;
  for (int k = 0; k < nc; ++k) {
    const uint32_t c = ld32(d, cig + 4ll * k), o = c & 15u;
    if (o == 4) start += c >> 4; else if (o != 5) break;
  }
  for (int k = nc - 1; k >= 1; --k) {
    const uint32_t c = ld32(d, cig + 4ll * k), o = c & 15u;
    if (o == 4) end -= c >> 4; else if (o != 5) break;
  }
  return end - start;
}

// The NM field of the auxiliary data [a, e): SC_OK with its type in *ty and, for a fixed-size type, its value's position
// in *at (the bytes are inside [a, e)); SC_NO_NM absent; SC_AUX malformed (before or at NM).
__device__ int locate_nm(const uint8_t *d, int64_t a, int64_t e, uint8_t *ty_out, int64_t *at) {
  while (a < e) {
    if (e - a < 3) return SC_AUX;
    const uint8_t t0 = d[a], t1 = d[a + 1], ty = d[a + 2];
    const bool is_nm = t0 == 'N' && t1 == 'M';
    a += 3;
    int sz = 0;
    switch (ty) {
      case 'A': case 'c': case 'C': sz = 1; break;
      case 's': case 'S': sz = 2; break;
      case 'i': case 'I': case 'f': sz = 4; break;
      case 'Z': case 'H': {
        int64_t z = a;
        while (z < e && d[z] != 0) ++z;
        if (z >= e) return SC_AUX;
        if (is_nm) { *ty_out = ty; return SC_OK; }
        a = z + 1;
        continue;
      }
      case 'B': {
        if (e - a < 5) return SC_AUX;
        const uint8_t st = d[a];
        const int es = (st == 'c' || st == 'C') ? 1 : (st == 's' || st == 'S') ? 2 : (st == 'i' || st == 'I' || st == 'f') ? 4 : 0;
        if (!es) return SC_AUX;
        const int64_t cnt = (int64_t)ld32(d, a + 1);
        if (cnt * es > e - a - 5) return SC_AUX;
        if (is_nm) { *ty_out = ty; return SC_OK; }
        a += 5 + cnt * es;
        continue;
      }
      default: return SC_AUX;
    }
    if (e - a < sz) return SC_AUX;
    if (is_nm) { *ty_out = ty; *at = a; return SC_OK; }
    a += sz;
  }
  return SC_NO_NM;
}

// an integer aux value of type cCsSiI at d[a]; false for any other type
__device__ __forceinline__ bool aux_int(const uint8_t *d, int64_t a, uint8_t ty, int64_t *v) {
  switch (ty) {
    case 'c': *v = (int8_t)d[a]; return true;
    case 'C': *v = d[a]; return true;
    case 's': *v = (int16_t)(d[a] | d[a + 1] << 8); return true;
    case 'S': *v = (uint16_t)(d[a] | d[a + 1] << 8); return true;
    case 'i': *v = (int32_t)ld32(d, a); return true;
    case 'I': *v = (uint32_t)ld32(d, a); return true;
    default: return false;
  }
}

// NM as an integer: 0 found, SC_NO_NM absent or not of type cCsSiI, SC_AUX malformed
__device__ int find_nm(const uint8_t *d, int64_t a, int64_t e, int64_t *nm) {
  uint8_t ty = 0;
  int64_t at = 0;
  const int rc = locate_nm(d, a, e, &ty, &at);
  if (rc) return rc;
  return aux_int(d, at, ty, nm) ? SC_OK : SC_NO_NM;
}

// NM as pysam's get_tag gives it to a numeric comparison: an integer type, or the float of type f (widened to double).
// 0 found, SC_NO_NUM_NM absent or of type A, Z, H or B, SC_AUX malformed.
__device__ int find_nm_number(const uint8_t *d, int64_t a, int64_t e, double *nm) {
  uint8_t ty = 0;
  int64_t at = 0;
  const int rc = locate_nm(d, a, e, &ty, &at);
  if (rc) return rc == SC_NO_NM ? SC_NO_NUM_NM : rc;
  int64_t v;
  if (aux_int(d, at, ty, &v)) { *nm = (double)v; return SC_OK; }
  if (ty == 'f') { *nm = (double)__uint_as_float(ld32(d, at)); return SC_OK; }
  return SC_NO_NUM_NM;
}

// One record's fields, decoded and bounds-checked by decode_record.
struct Rec {
  int32_t ref, pos, l_seq;
  int mapq, n_cigar, flag;
  int64_t cig, aux, end;                      // CIGAR and auxiliary data positions, the next record's position
};

// The record at stream position p of a segment ending at `end`: SC_OK, SC_TAIL at the first unplaced record of the last
// segment, or the code that stops the walk.
__device__ __forceinline__ int decode_record(const uint8_t *d, int64_t p, int64_t end, int32_t n_ref, bool last_seg, Rec &r) {
  if (end - p < 36) return SC_ANCHOR;
  const int32_t bs = (int32_t)ld32(d, p);
  if (bs < 32) return SC_RECORD;
  if (bs > end - p - 4) return SC_ANCHOR;
  r.ref = (int32_t)ld32(d, p + 4);
  if (r.ref < -1 || r.ref >= n_ref) return SC_REFID;
  if (r.ref == -1) return last_seg ? SC_TAIL : SC_UNPLACED;
  r.pos = (int32_t)ld32(d, p + 8);
  const uint32_t w3 = ld32(d, p + 12), w4 = ld32(d, p + 16);
  const int l_name = (int)(w3 & 0xFF);
  r.mapq = (int)((w3 >> 8) & 0xFF);
  r.n_cigar = (int)(w4 & 0xFFFF); r.flag = (int)(w4 >> 16);
  r.l_seq = (int32_t)ld32(d, p + 20);
  r.end = p + 4 + bs;
  r.cig = p + 4 + 32 + l_name;
  r.aux = r.cig + 4ll * r.n_cigar + ((int64_t)r.l_seq + 1) / 2 + r.l_seq;
  if (l_name < 1 || r.l_seq < 0 || r.aux > r.end) return SC_RECORD;
  return SC_OK;
}

__device__ __forceinline__ void flush(unsigned long long *counters, int ref, unsigned long long *c) {
  if (ref >= 0) {
    unsigned long long *dst = counters + (size_t)ref * NCNT;
#pragma unroll
    for (int k = 0; k < NCNT; ++k)
      if (c[k]) atomicAdd(dst + k, c[k]);
  }
#pragma unroll
  for (int k = 0; k < NCNT; ++k) c[k] = 0;
}

// The walk of one segment by one thread, shared by both kernels.  The counters stay in registers while refID is the same
// and are flushed when it changes; the walk ends at the segment's end, at the first unplaced record of the last segment,
// or at the first record that stops it, whose position goes into the error word.  What a record counts for is the rule's:
//   rule.reference(ref)     the walk enters reference ref (before its first record)
//   rule.record(d, r, c)    classifies the decoded record r into c: SC_OK, or the code that stops the walk at r
//   rule.finish()           after the final flush, whether or not the walk stopped early
template <class Rule>
__device__ __forceinline__ void walk(const WalkParams &q, Rule &rule) {
  const int64_t s = (int64_t)blockIdx.x * SCAN_THREADS + threadIdx.x;
  if (s >= q.nseg) return;
  const uint8_t *d = q.data;
  int64_t pos = q.seg_start[s];
  const int64_t end = q.seg_end[s];
  unsigned long long c[NCNT];
#pragma unroll
  for (int k = 0; k < NCNT; ++k) c[k] = 0;
  int cur = -1, code = SC_OK;
  while (pos < end) {
    Rec r;
    const int rc = decode_record(d, pos, end, q.n_ref, s == q.nseg - 1, r);
    if (rc) { if (rc != SC_TAIL) code = rc; break; }
    if (r.ref != cur) { flush(q.counters, cur, c); cur = r.ref; rule.reference(cur); }
    if ((code = rule.record(d, r, c))) break;
    pos = r.end;
  }
  if (code) atomicMin(q.err, (unsigned long long)pos << 8 | (unsigned long long)code);
  flush(q.counters, cur, c);
  rule.finish();
}

// coverage.py:206-230
struct CoverageRule {
  const ckm_bam_filter &f;
  __device__ void reference(int) {}
  __device__ int record(const uint8_t *d, const Rec &r, unsigned long long *c) const {
    const int flag = r.flag, l_seq = r.l_seq;
    c[0]++;
    if (flag & 0x4) {
    } else if (flag & 0x400) c[1]++;
    else if (flag & 0x900) c[2]++;
    else if ((flag & 0x200) || r.mapq < f.min_qc) c[3]++;
    else {
      const int64_t qal = aligned_length(d, r.cig, r.n_cigar, l_seq);
      if ((double)qal < f.min_align * (double)l_seq) c[4]++;
      else {
        int64_t nm = 0;
        const int rc = find_nm(d, r.aux, r.end, &nm);
        if (rc) return rc;
        if ((double)nm > f.max_edit * (double)l_seq) c[5]++;
        else if (!f.all_reads && !(flag & 0x2)) c[6]++;
        else { c[7]++; c[8] += (unsigned long long)qal; }
      }
    }
    return SC_OK;
  }
  __device__ void finish() {}
};

__global__ void __launch_bounds__(SCAN_THREADS) bam_scan_kernel(WalkParams q) {
  CoverageRule rule{q.filter};
  walk(q, rule);
}

struct WinParams {
  WalkParams walk;                            // counters: the ninth is the clipped covered bases
  const int64_t *ref_len;                     // header lengths
  const int64_t *win_off;                     // n_ref + 1: reference r's windows are windows[win_off[r] .. win_off[r + 1])
  int64_t W;
  unsigned long long *windows;                // per window: the sum of the depth over it
  unsigned long long *touched;                // [0] smallest window written, [1] largest + 1
};

// reference span of the CIGAR: M, D, N, =, X (pysam's reference_length, coverageWindows' `alen`)
__device__ __forceinline__ int64_t reference_span(const uint8_t *d, int64_t cig, int nc) {
  int64_t s = 0;
  for (int k = 0; k < nc; ++k) {
    const uint32_t c = ld32(d, cig + 4ll * k), o = c & 15u;
    if (o == 0 || o == 2 || o == 3 || o == 7 || o == 8) s += c >> 4;
  }
  return s;
}

// coverageWindows.py:55-79 over the records fetch(ref, 0, L) yields
struct WindowRule {
  const WinParams &q;
  int64_t L = 0, off = 0, nwin = 0;           // the current reference's length, first window and window count
  int64_t wi = -1;                            // cached window (global index) and its partial sum
  unsigned long long wsum = 0;
  unsigned long long lo = ~0ull, hi = 0;      // the windows written: [lo, hi)
  __device__ void reference(int ref) { L = q.ref_len[ref]; off = q.win_off[ref]; nwin = q.win_off[ref + 1] - off; }
  __device__ int record(const uint8_t *d, const Rec &r, unsigned long long *c) {
    const ckm_bam_filter &f = q.walk.filter;
    const int64_t W = q.W;
    const int flag = r.flag;
    const double l_seq = (double)r.l_seq;
    const int64_t alen = reference_span(d, r.cig, r.n_cigar);
    const int64_t rp = r.pos;
    // fetch(ref, 0, L) yields the records overlapping [0, L): end = pos + span, or pos + 1 when unmapped or empty
    const int64_t fend = rp + ((flag & 0x4) || alen == 0 ? 1 : alen);
    if (rp >= L || fend <= 0) return SC_OK;
    c[0]++;
    if (flag & 0x4) {
    } else if (flag & 0x400) c[1]++;
    else if (flag & 0x100) c[2]++;                                 // supplementary reads fall through
    else if (flag & 0x200) c[3]++;                                 // no mapping-quality threshold
    else if (r.n_cigar == 0) return SC_NO_CIGAR;
    else if ((double)alen < f.min_align * l_seq) c[4]++;
    else {
      double nm = 0.0;
      const int rc = find_nm_number(d, r.aux, r.end, &nm);
      if (rc) return rc;
      if (nm > f.max_edit * l_seq) c[5]++;
      else if (!f.all_reads && !(flag & 0x2)) c[6]++;
      else if (rp < 0) return SC_NEG_POS;
      else {
        c[7]++;
        const int64_t b = min(rp + alen, L);                       // numpy's slice clips at the reference end
        if (b > rp) {
          c[8] += (unsigned long long)(b - rp);
          const int64_t klast = min((b - 1) / W, nwin - 1);
          for (int64_t k = rp / W; k <= klast; ++k) {
            const int64_t g = off + k;
            if (g != wi) {
              if (wsum) atomicAdd(q.windows + wi, wsum);
              wi = g; wsum = 0;
              lo = min(lo, (unsigned long long)g); hi = max(hi, (unsigned long long)g + 1);
            }
            wsum += (unsigned long long)(min(b, (k + 1) * W) - max(rp, k * W));
          }
        }
      }
    }
    return SC_OK;
  }
  __device__ void finish() {
    if (wsum) atomicAdd(q.windows + wi, wsum);
    if (hi) { atomicMin(q.touched, lo); atomicMax(q.touched + 1, hi); }
  }
};

__global__ void __launch_bounds__(SCAN_THREADS) bam_window_kernel(WinParams q) {
  WindowRule rule{q};
  walk(q.walk, rule);
}

const uint32_t *x2n_table() {
  static uint32_t t[32];
  static bool done = false;
  if (!done) {
    auto mul = [](uint32_t a, uint32_t b) {
      uint32_t m = 1u << 31, p = 0;
      for (;;) {
        if (a & m) { p ^= b; if ((a & (m - 1)) == 0) break; }
        m >>= 1;
        b = b & 1 ? (b >> 1) ^ CRC_POLY : b >> 1;
      }
      return p;
    };
    uint32_t p = 1u << 30;                                         // x^1
    t[0] = p;
    for (int k = 1; k < 32; ++k) t[k] = p = mul(p, p);
    done = true;
  }
  return t;
}

// Checks the block table against the compressed range and fills the exclusive prefix sum of ISIZE.
int check_blocks(const char *fn, int64_t comp_base, int64_t comp_len, const ckm_bgzf_block *blocks, int64_t nblocks,
                 std::vector<int64_t> &uoff) {
  uoff.resize((size_t)nblocks + 1);
  int64_t u = 0;
  for (int64_t b = 0; b < nblocks; ++b) {
    const ckm_bgzf_block &k = blocks[b];
    const int64_t rel = k.coffset - comp_base;
    if (rel < 0 || k.clen < 26 || k.clen > 65536 || rel + k.clen > comp_len || k.isize < 0 || k.isize > 65536) {
      char msg[192];
      std::snprintf(msg, sizeof msg, "%s: block %lld (file offset %lld) does not lie in the compressed range or has a bad size",
                    fn, (long long)b, (long long)k.coffset);
      set_error(msg); return CKM_EINVAL;
    }
    uoff[b] = u; u += k.isize;
  }
  uoff[nblocks] = u;
  return CKM_OK;
}

// Uploads the batch and inflates it into dout (uoff.back() bytes + 8 of zero padding).  On a bad block: CKM_EFORMAT, the
// message names the block's file offset, *bad_block_out its index.
int inflate_batch(ckm_engine *e, const char *fn, const uint8_t *comp, int64_t comp_base, int64_t comp_len,
                  const ckm_bgzf_block *blocks, int64_t nblocks, const std::vector<int64_t> &uoff, DevBuf &dout,
                  int64_t *bad_block_out, float *ms_out) {
  cudaStream_t st = e->stream;
  const int64_t total = uoff.back();
  DevBuf dcomp, dblk, duoff, dstat, dbad;
  CKM_TRY(dcomp.put(comp, (size_t)comp_len, st));
  CKM_TRY(dblk.put(blocks, (size_t)nblocks, st));
  CKM_TRY(duoff.put(uoff.data(), uoff.size(), st));
  CKM_TRY(dstat.alloc(sizeof(int) * (size_t)nblocks));
  CKM_TRY(dbad.fill(sizeof(unsigned long long), 0xFF, st));
  CKM_TRY(dout.alloc((size_t)total + 16));
  CKM_TRY(set_bytes(dout.as<uint8_t>() + total, 0, 16, st));
  InflateParams p;
  p.comp = dcomp.as<uint8_t>(); p.comp_base = comp_base;
  p.blocks = dblk.as<ckm_bgzf_block>(); p.uoff = duoff.as<int64_t>(); p.nblocks = nblocks;
  p.out = dout.as<uint8_t>(); p.status = dstat.as<int>(); p.first_bad = dbad.as<unsigned long long>();
  std::memcpy(p.x2n, x2n_table(), sizeof(p.x2n));
  CKM_TRY(ev_record(e, 0));
  if (nblocks) {
    bgzf_inflate_kernel<<<(unsigned)((nblocks + IW - 1) / IW), IW * 32, 0, st>>>(p);
    CKM_CUDA(cudaGetLastError());
  }
  CKM_TRY(ev_record(e, 1));
  unsigned long long bad = 0;
  CKM_TRY(dbad.get(&bad, 1, st));
  CKM_TRY(stream_sync(st));
  CKM_TRY(ev_elapsed(e, ms_out, 0, 1));
  if (bad != ~0ull) {
    int code = 0;
    CKM_TRY(dstat.get(&code, 1, st, bad));
    CKM_TRY(stream_sync(st));
    char msg[256];
    std::snprintf(msg, sizeof msg, "%s: BGZF block at file offset %lld: %s", fn, (long long)blocks[bad].coffset, inflate_msg(code));
    set_error(msg);
    if (bad_block_out) *bad_block_out = (int64_t)bad;
    return CKM_EFORMAT;
  }
  return CKM_OK;
}

// check_blocks, and every segment inside the batch's decompressed range
int check_batch(const char *fn, int64_t comp_base, int64_t comp_len, const ckm_bgzf_block *blocks, int64_t nblocks,
                const int64_t *seg_start, const int64_t *seg_end, int64_t nseg, std::vector<int64_t> &uoff) {
  int rc;
  if ((rc = check_blocks(fn, comp_base, comp_len, blocks, nblocks, uoff))) return rc;
  const int64_t total = uoff.back();
  for (int64_t s = 0; s < nseg; ++s)
    if (seg_start[s] < 0 || seg_start[s] > seg_end[s] || seg_end[s] > total) {
      char msg[160];
      std::snprintf(msg, sizeof msg, "%s: a segment does not lie in the batch's decompressed range", fn);
      set_error(msg); return CKM_EINVAL;
    }
  return CKM_OK;
}

// CKM_EFORMAT for a walk's error word (record position << 8 | code): the record's virtual offset and, for the codes
// that concern one read, its name.
int scan_error(const char *fn, unsigned long long err, const ckm_bgzf_block *blocks, int64_t nblocks,
               const std::vector<int64_t> &uoff, DevBuf &dout, int64_t *err_offset_out) {
  const int64_t total = uoff.back();
  const int code = (int)(err & 0xFF);
  const int64_t pos = (int64_t)(err >> 8);
  const int64_t b = std::upper_bound(uoff.begin(), uoff.end() - 1, pos) - uoff.begin() - 1;   // block holding pos
  const int64_t voff = b >= 0 && b < nblocks ? (blocks[b].coffset << 16 | (pos - uoff[b])) : -1;
  std::string name;
  if (scan_names_read(code)) {
    char rec[300];
    const int64_t nb = std::min<int64_t>((int64_t)sizeof rec, total + 8 - pos);
    CKM_CUDA(cudaMemcpy(rec, dout.as<uint8_t>() + pos, (size_t)nb, cudaMemcpyDeviceToHost));
    const int l = (uint8_t)rec[12];
    for (int i = 0; i < l - 1 && 36 + i < nb && rec[36 + i]; ++i) name += rec[36 + i];
  }
  char msg[512];
  std::snprintf(msg, sizeof msg, "%s: record at virtual offset %lld (block at file offset %lld + %lld): %s%s%s", fn,
                (long long)voff, (long long)(b >= 0 && b < nblocks ? blocks[b].coffset : -1), (long long)(b >= 0 ? pos - uoff[b] : -1),
                scan_msg(code), name.empty() ? "" : " in read ", name.c_str());
  set_error(msg);
  if (err_offset_out) *err_offset_out = voff;
  return CKM_EFORMAT;
}

struct NoStep { int operator()() const { return CKM_OK; } };

// One batch of ckm_bam_coverage or ckm_bam_windows (fn), from the argument check to the sum into `counters`: the batch
// checks, the inflate, the segments, counters and error word on the device, the walk timed by events and its error.
// launch(q, grid, st) launches the walk kernel with the shared parameters q.  prepare() runs after the batch checks and
// before the inflate, in the same pool scope as the walk: the caller's own checks and buffers.  finish() runs after a
// walk without error.
template <class Launch, class Prepare = NoStep, class Finish = NoStep>
int walk_batch(const char *fn, ckm_engine *e, const uint8_t *comp, int64_t comp_base, int64_t comp_len,
               const ckm_bgzf_block *blocks, int64_t nblocks, const int64_t *seg_start, const int64_t *seg_end, int64_t nseg,
               int32_t n_ref, const ckm_bam_filter *filter, int64_t *counters, float *kernel_ms_out, int64_t *err_offset_out,
               Launch launch, Prepare prepare = Prepare(), Finish finish = Finish()) {
  if (!e || comp_len < 0 || (comp_len > 0 && !comp) || nblocks < 0 || (nblocks > 0 && !blocks) || nseg < 0 ||
      (nseg > 0 && (!seg_start || !seg_end)) || n_ref < 0 || !filter || (n_ref > 0 && !counters)) {
    set_error(std::string(fn) + ": bad argument"); return CKM_EINVAL;
  }
  if (kernel_ms_out) kernel_ms_out[0] = kernel_ms_out[1] = 0.0f;
  if (err_offset_out) *err_offset_out = -1;
  std::vector<int64_t> uoff;
  int rc;
  if ((rc = check_batch(fn, comp_base, comp_len, blocks, nblocks, seg_start, seg_end, nseg, uoff))) return rc;
  const DeviceScope ws(e);
  if ((rc = prepare())) return rc;
  DevBuf dout, dseg, dcnt, derr;
  int64_t bad_block = -1;
  float ms_inflate = 0.0f;
  if ((rc = inflate_batch(e, fn, comp, comp_base, comp_len, blocks, nblocks, uoff, dout, &bad_block, &ms_inflate))) {
    if (err_offset_out && bad_block >= 0) *err_offset_out = blocks[bad_block].coffset;
    return rc;
  }
  if (kernel_ms_out) kernel_ms_out[0] = ms_inflate;
  const size_t ncnt = (size_t)n_ref * NCNT;
  CKM_TRY(dseg.alloc(sizeof(int64_t) * 2 * (size_t)nseg));
  CKM_TRY(copy_in(dseg.as<int64_t>(), seg_start, (size_t)nseg, ws.st));
  CKM_TRY(copy_in(dseg.as<int64_t>() + nseg, seg_end, (size_t)nseg, ws.st));
  CKM_TRY(dcnt.fill(sizeof(int64_t) * ncnt, 0, ws.st));
  CKM_TRY(derr.fill(sizeof(unsigned long long), 0xFF, ws.st));
  WalkParams q;
  q.data = dout.as<uint8_t>(); q.seg_start = dseg.as<int64_t>(); q.seg_end = dseg.as<int64_t>() + nseg; q.nseg = nseg;
  q.n_ref = n_ref; q.filter = *filter;
  q.counters = dcnt.as<unsigned long long>(); q.err = derr.as<unsigned long long>();
  CKM_TRY(ev_record(e, 0));
  if (nseg) {
    launch(q, (unsigned)((nseg + SCAN_THREADS - 1) / SCAN_THREADS), ws.st);
    CKM_CUDA(cudaGetLastError());
  }
  CKM_TRY(ev_record(e, 1));
  unsigned long long err = 0;
  std::vector<int64_t> cnt(ncnt);
  CKM_TRY(derr.get(&err, 1, ws.st));
  CKM_TRY(dcnt.get(cnt.data(), ncnt, ws.st));
  CKM_TRY(stream_sync(ws.st));
  float ms_scan = 0.0f;
  CKM_TRY(ev_elapsed(e, &ms_scan, 0, 1));
  if (kernel_ms_out) kernel_ms_out[1] = ms_scan;
  if (err != ~0ull) return scan_error(fn, err, blocks, nblocks, uoff, dout, err_offset_out);
  for (size_t k = 0; k < ncnt; ++k) counters[k] += cnt[k];
  return finish();
}

}  // namespace

extern "C" {

int ckm_bgzf_blocks(const uint8_t *data, int64_t n, int64_t base, ckm_bgzf_block *blocks_out, int64_t cap,
                    int64_t *nblocks_out, int64_t *consumed_out) {
  static_assert(sizeof(ckm_bgzf_block) == 16, "ckm_bgzf_block is 16 bytes");
  if (n < 0 || (n > 0 && !data) || cap < 0 || (cap > 0 && !blocks_out) || !nblocks_out || !consumed_out) {
    set_error("ckm_bgzf_blocks: bad argument"); return CKM_EINVAL;
  }
  int64_t p = 0, k = 0;
  auto bad = [&](const char *why) {
    char msg[192];
    std::snprintf(msg, sizeof msg, "ckm_bgzf_blocks: not a BGZF block at file offset %lld (%s)", (long long)(base + p), why);
    set_error(msg);
    *nblocks_out = k; *consumed_out = p;
    return (int)CKM_EFORMAT;
  };
  while (k < cap && n - p >= 12) {
    const uint8_t *h = data + p;
    if (h[0] != 0x1f || h[1] != 0x8b || h[2] != 8 || h[3] != 4) return bad("gzip magic 1f 8b 08 04 expected");
    const int xlen = h[10] | h[11] << 8;
    if (n - p < 12 + xlen) break;                                  // header not wholly inside the range
    int bsize = -1, q = 12;
    while (q + 4 <= 12 + xlen) {
      const int slen = h[q + 2] | h[q + 3] << 8;
      if (h[q] == 'B' && h[q + 1] == 'C' && slen == 2 && q + 6 <= 12 + xlen) bsize = h[q + 4] | h[q + 5] << 8;
      q += 4 + slen;
    }
    if (q != 12 + xlen) return bad("extra subfields overrun XLEN");
    if (bsize < 0) return bad("no BC subfield");
    const int64_t blen = (int64_t)bsize + 1;
    if (blen < 12 + xlen + 8) return bad("BSIZE smaller than its header and trailer");
    if (p + blen > n) break;                                       // block not wholly inside the range
    const uint8_t *t = h + blen - 4;
    const uint32_t isize = (uint32_t)t[0] | (uint32_t)t[1] << 8 | (uint32_t)t[2] << 16 | (uint32_t)t[3] << 24;
    if (isize > 65536) return bad("ISIZE above 64 KiB");
    blocks_out[k].coffset = base + p; blocks_out[k].clen = (int32_t)blen; blocks_out[k].isize = (int32_t)isize;
    ++k; p += blen;
  }
  *nblocks_out = k; *consumed_out = p;
  return CKM_OK;
}

int ckm_bgzf_inflate(ckm_engine *e, const uint8_t *comp, int64_t comp_base, int64_t comp_len, const ckm_bgzf_block *blocks,
                     int64_t nblocks, uint8_t *out, int64_t out_cap, int64_t *bad_block_out, float *kernel_ms_out) {
  if (!e || comp_len < 0 || (comp_len > 0 && !comp) || nblocks < 0 || (nblocks > 0 && !blocks) || out_cap < 0 ||
      (out_cap > 0 && !out)) {
    set_error("ckm_bgzf_inflate: bad argument"); return CKM_EINVAL;
  }
  if (bad_block_out) *bad_block_out = -1;
  if (kernel_ms_out) *kernel_ms_out = 0.0f;
  std::vector<int64_t> uoff;
  int rc;
  if ((rc = check_blocks("ckm_bgzf_inflate", comp_base, comp_len, blocks, nblocks, uoff))) return rc;
  if (uoff.back() > out_cap) { set_error("ckm_bgzf_inflate: output buffer smaller than the sum of ISIZE"); return CKM_ECAPACITY; }
  const DeviceScope ws(e);
  DevBuf dout;
  float ms = 0.0f;
  if ((rc = inflate_batch(e, "ckm_bgzf_inflate", comp, comp_base, comp_len, blocks, nblocks, uoff, dout, bad_block_out, &ms)))
    return rc;
  if (kernel_ms_out) *kernel_ms_out = ms;
  CKM_TRY(dout.get(out, (size_t)uoff.back(), ws.st));
  return stream_sync(ws.st);
}

int ckm_bam_coverage(ckm_engine *e, const uint8_t *comp, int64_t comp_base, int64_t comp_len, const ckm_bgzf_block *blocks,
                     int64_t nblocks, const int64_t *seg_start, const int64_t *seg_end, int64_t nseg, int32_t n_ref,
                     const ckm_bam_filter *filter, int64_t *counters, float *kernel_ms_out, int64_t *err_offset_out) {
  return walk_batch("ckm_bam_coverage", e, comp, comp_base, comp_len, blocks, nblocks, seg_start, seg_end, nseg, n_ref, filter,
                    counters, kernel_ms_out, err_offset_out,
                    [](const WalkParams &q, unsigned grid, cudaStream_t st) { bam_scan_kernel<<<grid, SCAN_THREADS, 0, st>>>(q); });
}

int ckm_bam_windows(ckm_engine *e, const uint8_t *comp, int64_t comp_base, int64_t comp_len, const ckm_bgzf_block *blocks,
                    int64_t nblocks, const int64_t *seg_start, const int64_t *seg_end, int64_t nseg, int32_t n_ref,
                    const ckm_bam_filter *filter, const int64_t *ref_len, int64_t window_size, const int64_t *win_off,
                    int64_t *counters, int64_t *windows, float *kernel_ms_out, int64_t *err_offset_out) {
  DevBuf dwin, dlen, dtouch;
  auto prepare = [&]() -> int {
    if ((n_ref > 0 && !ref_len) || !win_off) { set_error("ckm_bam_windows: bad argument"); return CKM_EINVAL; }
    char msg[320];
    if (window_size <= 0) {
      std::snprintf(msg, sizeof msg, "ckm_bam_windows: window size %lld; it must be at least 1", (long long)window_size);
      set_error(msg); return CKM_EINVAL;
    }
    if (win_off[0] != 0) { set_error("ckm_bam_windows: win_off[0] must be 0"); return CKM_EINVAL; }
    for (int32_t r = 0; r < n_ref; ++r) {
      if (ref_len[r] <= 0) {
        std::snprintf(msg, sizeof msg, "ckm_bam_windows: reference %d has length %lld; coverage per base needs a length of at "
                      "least 1", r, (long long)ref_len[r]);
        set_error(msg); return CKM_EINVAL;
      }
      if (win_off[r + 1] - win_off[r] != (ref_len[r] - 1) / window_size) {
        std::snprintf(msg, sizeof msg, "ckm_bam_windows: reference %d has %lld windows in win_off, (length - 1) / window size "
                      "is %lld", r, (long long)(win_off[r + 1] - win_off[r]), (long long)((ref_len[r] - 1) / window_size));
        set_error(msg); return CKM_EINVAL;
      }
    }
    const int64_t nwin = win_off[n_ref];
    if (nwin > 0 && !windows) { set_error("ckm_bam_windows: bad argument"); return CKM_EINVAL; }
    // the window array first: it is the one buffer whose size the caller chooses through W
    size_t free_b = 0, total_b = 0;
    CKM_CUDA(cudaMemGetInfo(&free_b, &total_b));
    const double need = 8.0 * (double)nwin;
    if (need > (double)free_b || dwin.alloc(sizeof(int64_t) * (size_t)nwin)) {
      cudaGetLastError();
      if (need <= (double)free_b) CKM_CUDA(cudaMemGetInfo(&free_b, &total_b));
      // the smallest W whose window array fits in the free memory (sum of (len - 1) / W falls as W grows)
      auto windows_at = [&](int64_t w) { int64_t t = 0; for (int32_t r = 0; r < n_ref; ++r) t += (ref_len[r] - 1) / w; return t; };
      const int64_t cap = (int64_t)(free_b / 8);
      int64_t lo_w = window_size, hi_w = window_size;
      while (windows_at(hi_w) > cap && hi_w < (int64_t(1) << 40)) hi_w *= 2;
      while (lo_w < hi_w) { const int64_t m = lo_w + (hi_w - lo_w) / 2; if (windows_at(m) > cap) lo_w = m + 1; else hi_w = m; }
      std::snprintf(msg, sizeof msg, "ckm_bam_windows: %lld windows of %lld bp need %.1f MiB of device memory, %.1f MiB are "
                    "free; the smallest window size that fits is %lld", (long long)nwin, (long long)window_size,
                    need / 1048576.0, (double)free_b / 1048576.0, (long long)lo_w);
      set_error(msg); return CKM_ENOMEM;
    }
    cudaStream_t st = e->stream;
    CKM_TRY(set_bytes(dwin.p, 0, sizeof(int64_t) * (size_t)nwin, st));
    const unsigned long long touched0[2] = {~0ull, 0ull};
    CKM_TRY(dtouch.put(touched0, 2, st));
    CKM_TRY(dlen.alloc(sizeof(int64_t) * (2 * (size_t)n_ref + 1)));
    CKM_TRY(copy_in(dlen.as<int64_t>(), ref_len, (size_t)n_ref, st));
    return copy_in(dlen.as<int64_t>() + n_ref, win_off, (size_t)n_ref + 1, st);
  };
  auto launch = [&](const WalkParams &w, unsigned grid, cudaStream_t st) {
    const WinParams q{w, dlen.as<int64_t>(), dlen.as<int64_t>() + n_ref, window_size, dwin.as<unsigned long long>(),
                      dtouch.as<unsigned long long>()};
    bam_window_kernel<<<grid, SCAN_THREADS, 0, st>>>(q);
  };
  // only the windows this batch wrote come back: a batch covers a run of references, not the whole array
  auto finish = [&]() -> int {
    unsigned long long touched[2];
    CKM_TRY(dtouch.get(touched, 2, e->stream));
    CKM_TRY(stream_sync(e->stream));
    if (touched[1] > touched[0]) {
      const size_t lo = (size_t)touched[0], n = (size_t)(touched[1] - touched[0]);
      std::vector<int64_t> w(n);
      CKM_TRY(dwin.get(w.data(), n, e->stream, lo));
      CKM_TRY(stream_sync(e->stream));
      for (size_t k = 0; k < n; ++k) windows[lo + k] += w[k];
    }
    return CKM_OK;
  };
  return walk_batch("ckm_bam_windows", e, comp, comp_base, comp_len, blocks, nblocks, seg_start, seg_end, nseg, n_ref, filter,
                    counters, kernel_ms_out, err_offset_out, launch, prepare, finish);
}

}  // extern "C"
