// FLAC decoding of a packed ragged batch of streams (ttsb_flac_decode_batch): the decoding half of librosa.load on a .flac file
// (libsndfile -> float32, then the mono mix-down), as the reference's Audio.load_wav reaches it (reference: data/audio.py:126-130).
// The format is RFC 9639; the host parses the metadata blocks (data/audio.py: read_flac_info) and passes the frame bytes of every
// file, concatenated, with each file's STREAMINFO.
//
// Five launches per batch whatever the number of files:
//   1. find   (one CTA per file, one thread per byte position): every position that holds a well-formed frame header of the
//             file's blocking strategy with a matching CRC-8 is a candidate; a block-wide ballot scan compacts the candidates of
//             the file in byte order (no atomics).  Two candidates are at least 5 bytes apart (bytes 1..4 of a header cannot be
//             0xFF), so a file of L bytes has at most ceil(L / 5).
//   2. parse  (one thread per candidate): reads every subframe without storing it, the zero padding and the CRC-16, and records
//             where the frame ends and whether it is well formed.  A candidate whose header disagrees with STREAMINFO is not parsed.
//   3. chain  (one thread per file): the real frames are the first frame and each candidate at which a real frame ends; the walk
//             checks the coded frame number (fixed blocking) or sample number (variable blocking), the header against STREAMINFO
//             and the total, and writes the frame table.  A sync pattern inside subframe data is never on the chain.
//   4. decode (one thread per (frame, channel)): skips the frame's earlier subframes and decodes its own into the file's planar
//             int32 PCM: CONSTANT, VERBATIM, FIXED 0-4, LPC 1-32, Rice / Rice2 residuals with escapes, int64 prediction, the
//             wasted-bits shift.
//   5. output (one thread per output sample): undoes the stereo decorrelation, scales by 2^-(bps - 1) as libsndfile does and mixes
//             down to mono in numpy's order for np.mean(y, axis=1) on float32: ((x0 + x1) + x2) + ... for up to 7 channels, the
//             pairwise ((x0 + x1) + (x2 + x3)) + ((x4 + x5) + (x6 + x7)) for 8, then an IEEE division by the channel count.
//
// Every read of the bit reader is bounded by the file's byte range, so a corrupt stream gives a status and never a load outside
// it.  The MD5 of STREAMINFO is not checked (libsndfile does not check it either).
#include <limits.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "../../include/ttsb.h"
#include "ttsb_common.cuh"
#include "ttsb_host.h"

namespace ttsb {
namespace {

constexpr int FLAC_FIND_THREADS = 512;
constexpr int FLAC_THREADS = 128;
constexpr int FLAC_MAX_LPC = 32;

struct FlacFile {          // per file; written by the host
  int64_t byte_start;      // its frame bytes: data[byte_start .. byte_start + byte_len)
  int64_t total;           // STREAMINFO's samples per channel
  int64_t cand_base;       // its first candidate slot
  int64_t frame_base;      // its first frame-table slot
  int64_t plane_base;      // its planar PCM in the workspace, channel c at plane_base + c total
  int64_t mono_base;       // its first sample in mono_out
  int64_t pcm_base;        // its first value in pcm_out (interleaved)
  int32_t byte_len, frame_cap;
  int32_t channels, bps, rate, min_block, max_block;
};

struct FlacHeader {
  int32_t len;             // header bytes, CRC-8 included
  int32_t block;           // samples per channel
  int32_t rate;            // Hz (the STREAMINFO rate for code 0)
  int32_t assign;          // channel assignment code 0..10
  int32_t channels;
  int32_t bps;             // bits per sample (the STREAMINFO depth for code 0)
  int64_t number;          // coded frame number (fixed blocking) or sample number (variable blocking)
};

struct FlacFrame {
  int64_t start;           // first sample of the frame in its file
  int32_t pos;             // header byte position in the file
  int32_t block;
  int32_t assign;
  int32_t pad;
};

__device__ __forceinline__ void flac_tables(uint8_t* crc8, uint16_t* crc16) {
  for (int i = threadIdx.x; i < 256; i += blockDim.x) {
    uint32_t c8 = (uint32_t)i, c16 = (uint32_t)i << 8;
    for (int k = 0; k < 8; ++k) {
      c8 = (c8 & 0x80u) ? ((c8 << 1) ^ 0x07u) : (c8 << 1);
      c16 = (c16 & 0x8000u) ? ((c16 << 1) ^ 0x8005u) : (c16 << 1);
    }
    if (crc8) crc8[i] = (uint8_t)c8;
    if (crc16) crc16[i] = (uint16_t)c16;
  }
}

// The frame header at f[pos] (f: the file's frame bytes, len of them), or false: sync 0xFFF8 | blocking, zero reserved bits, valid
// block-size / rate / channel / depth codes, a well-formed coded number (at most 31 bits for a frame number), the trailing block
// size and rate bytes, and the CRC-8 (polynomial 0x07) over the header.
__device__ __forceinline__ bool flac_header(const uint8_t* __restrict__ f, int len, int pos, int blocking, const FlacFile& fd,
                            const uint8_t* crc8, FlacHeader& h) {
  const int room = len - pos;
  if (room < 6) return false;
  const uint8_t* p = f + pos;
  if (__ldg(p) != 0xFF || __ldg(p + 1) != (0xF8 | blocking)) return false;
  const int b2 = __ldg(p + 2), b3 = __ldg(p + 3);
  const int bs_code = b2 >> 4, sr_code = b2 & 15, ch_code = b3 >> 4, bps_code = (b3 >> 1) & 7;
  if (bs_code == 0 || sr_code == 15 || ch_code > 10 || bps_code == 3 || (b3 & 1)) return false;
  int n = 4;
  const int lead = __ldg(p + n++);
  int extra;
  int64_t num;
  if (lead < 0x80) { num = lead; extra = 0; }
  else if (lead < 0xC0) return false;
  else if (lead < 0xE0) { num = lead & 0x1F; extra = 1; }
  else if (lead < 0xF0) { num = lead & 0x0F; extra = 2; }
  else if (lead < 0xF8) { num = lead & 0x07; extra = 3; }
  else if (lead < 0xFC) { num = lead & 0x03; extra = 4; }
  else if (lead < 0xFE) { num = lead & 0x01; extra = 5; }
  else if (lead == 0xFE) { num = 0; extra = 6; }
  else return false;
  if (extra == 6 && !blocking) return false;
  const int tail = (bs_code == 6) + 2 * (bs_code == 7) + (sr_code == 12) + 2 * (sr_code == 13 || sr_code == 14);
  if (room < n + extra + tail + 1) return false;
  for (int k = 0; k < extra; ++k) {
    const int c = __ldg(p + n++);
    if ((c & 0xC0) != 0x80) return false;
    num = (num << 6) | (c & 0x3F);
  }
  int block;
  if (bs_code == 1) block = 192;
  else if (bs_code <= 5) block = 576 << (bs_code - 2);
  else if (bs_code >= 8) block = 256 << (bs_code - 8);
  else if (bs_code == 6) block = __ldg(p + n++) + 1;
  else { block = ((__ldg(p + n) << 8) | __ldg(p + n + 1)) + 1; n += 2; }
  int rate;
  switch (sr_code) {
    case 0: rate = fd.rate; break;
    case 1: rate = 88200; break;
    case 2: rate = 176400; break;
    case 3: rate = 192000; break;
    case 4: rate = 8000; break;
    case 5: rate = 16000; break;
    case 6: rate = 22050; break;
    case 7: rate = 24000; break;
    case 8: rate = 32000; break;
    case 9: rate = 44100; break;
    case 10: rate = 48000; break;
    case 11: rate = 96000; break;
    case 12: rate = __ldg(p + n++) * 1000; break;
    case 13: rate = (__ldg(p + n) << 8) | __ldg(p + n + 1); n += 2; break;
    default: rate = ((__ldg(p + n) << 8) | __ldg(p + n + 1)) * 10; n += 2; break;
  }
  uint32_t crc = 0;
  for (int k = 0; k < n; ++k) crc = crc8[crc ^ __ldg(p + k)];
  if (crc != __ldg(p + n)) return false;
  h.len = n + 1;
  h.block = block;
  h.rate = rate;
  h.assign = ch_code;
  h.channels = ch_code < 8 ? ch_code + 1 : 2;
  h.bps = bps_code == 0 ? fd.bps : bps_code == 1 ? 8 : bps_code == 2 ? 12 : bps_code == 7 ? 32 : 16 + 4 * (bps_code - 4);
  h.number = num;
  return true;
}

// Length of a header that flac_header has accepted.
__device__ __forceinline__ int flac_header_len(const uint8_t* p) {
  const int b2 = __ldg(p + 2), lead = __ldg(p + 4);
  const int bs_code = b2 >> 4, sr_code = b2 & 15;
  const int extra = lead < 0x80 ? 0 : lead < 0xE0 ? 1 : lead < 0xF0 ? 2 : lead < 0xF8 ? 3 : lead < 0xFC ? 4 : lead < 0xFE ? 5 : 6;
  return 6 + extra + (bs_code == 6) + 2 * (bs_code == 7) + (sr_code == 12) + 2 * (sr_code == 13 || sr_code == 14);
}

// 64-bit MSB-first bit reader over one file's bytes; a read past the end sets `bad` and returns zeros from then on.
struct FlacBits {
  const uint8_t* f;
  int len, next, avail;
  uint64_t cache;          // the next `avail` bits, left-aligned; the bits below them are zero
  bool bad;

  __device__ void init(const uint8_t* f_, int len_, int byte) {
    f = f_; len = len_; next = byte; avail = 0; cache = 0; bad = false;
  }
  __device__ __forceinline__ void refill() {
    while (avail <= 56 && next < len) {
      cache |= (uint64_t)__ldg(f + next) << (56 - avail);
      ++next;
      avail += 8;
    }
  }
  __device__ __forceinline__ void fail() { bad = true; next = len; avail = 0; cache = 0; }
  __device__ __forceinline__ int64_t tell() const { return (int64_t)next * 8 - avail; }
  __device__ __forceinline__ uint32_t get(int n) {        // 0 <= n <= 32
    if (avail < n) {
      refill();
      if (avail < n) { fail(); return 0; }
    }
    if (n == 0) return 0;
    const uint32_t v = (uint32_t)(cache >> (64 - n));
    cache <<= n;
    avail -= n;
    return v;
  }
  __device__ __forceinline__ int32_t get_signed(int n) {  // 1 <= n <= 32
    return (int32_t)(get(n) << (32 - n)) >> (32 - n);
  }
  __device__ __forceinline__ uint32_t unary() {           // zeros before the next one bit
    uint32_t zeros = 0;
    for (;;) {
      if (avail == 0) {
        refill();
        if (avail == 0) { fail(); return 0; }
      }
      const int lz = __clzll((long long)cache);
      if (lz < avail) {
        cache = lz == 63 ? 0 : cache << (lz + 1);
        avail -= lz + 1;
        return zeros + (uint32_t)lz;
      }
      zeros += (uint32_t)avail;
      cache = 0;
      avail = 0;
    }
  }
};

__device__ __forceinline__ bool flac_side(int assign, int c) {
  return (assign == 8 && c == 1) || (assign == 9 && c == 0) || (assign == 10 && c == 1);
}

// Reads one subframe of `block` samples at `bits` bits (the frame depth, plus one for a side channel).  kStore: decodes it into
// out[0 .. block) with `coef` (FLAC_MAX_LPC ints, any memory) as scratch; else only advances the reader.  -> 0 or a TTSB_FLAC_*.
template <bool kStore>
__device__ __forceinline__ int flac_subframe(FlacBits& br, int block, int bits, int32_t* out, int32_t* coef, int coef_stride) {
  if (br.get(1) != 0) return TTSB_FLAC_BAD_FRAME;
  const int type = (int)br.get(6);
  int wasted = 0;
  if (br.get(1)) wasted = (int)br.unary() + 1;
  if (br.bad) return TTSB_FLAC_TRUNCATED;
  if (wasted >= bits) return TTSB_FLAC_BAD_FRAME;
  bits -= wasted;
  int order = 0;
  if (type == 0) {
    const int32_t v = br.get_signed(bits);
    if (br.bad) return TTSB_FLAC_TRUNCATED;
    if (kStore) for (int i = 0; i < block; ++i) out[i] = v;
  } else if (type == 1) {
    for (int i = 0; i < block && !br.bad; ++i) {
      const int32_t v = br.get_signed(bits);
      if (kStore) out[i] = v;
    }
    if (br.bad) return TTSB_FLAC_TRUNCATED;
  } else {
    const bool lpc = type >= 32;
    if (lpc) order = type - 31;
    else if (type >= 8 && type <= 12) order = type - 8;
    else return TTSB_FLAC_BAD_FRAME;
    if (order > block) return TTSB_FLAC_BAD_FRAME;
    for (int i = 0; i < order; ++i) {
      const int32_t v = br.get_signed(bits);
      if (kStore) out[i] = v;
    }
    int shift = 0;
    if (lpc) {
      const int prec = (int)br.get(4);
      if (prec == 15) return br.bad ? TTSB_FLAC_TRUNCATED : TTSB_FLAC_BAD_FRAME;
      shift = br.get_signed(5);
      if (br.bad) return TTSB_FLAC_TRUNCATED;
      if (shift < 0) return TTSB_FLAC_BAD_FRAME;
      for (int j = 0; j < order; ++j) {
        const int32_t c = br.get_signed(prec + 1);
        if (kStore) coef[j * coef_stride] = c;
      }
    }
    // residual: Rice (4-bit parameters, escape 1111) or Rice2 (5-bit, escape 11111), 2^porder partitions
    const int method = (int)br.get(2);
    const int porder = (int)br.get(4);
    if (br.bad) return TTSB_FLAC_TRUNCATED;
    if (method > 1) return TTSB_FLAC_BAD_FRAME;
    if (block & ((1 << porder) - 1)) return TTSB_FLAC_BAD_FRAME;
    const int psize = block >> porder;
    if (psize < order) return TTSB_FLAC_BAD_FRAME;
    const int pbits = method ? 5 : 4, escape = method ? 31 : 15;
    int i = order;
    for (int part = 0; part < (1 << porder); ++part) {
      const int n = part ? psize : psize - order;
      const int k = (int)br.get(pbits);
      if (k == escape) {
        const int w = (int)br.get(5);
        for (int j = 0; j < n && !br.bad; ++j) {
          const int32_t r = w ? br.get_signed(w) : 0;
          if (kStore) out[i + j] = r;
        }
      } else {
        for (int j = 0; j < n && !br.bad; ++j) {
          const uint32_t q = br.unary();
          const uint32_t lo = br.get(k);
          const uint64_t u = ((uint64_t)q << k) | lo;
          const int64_t r = (int64_t)(u >> 1) ^ -(int64_t)(u & 1);
          if (kStore) out[i + j] = (int32_t)r;
        }
      }
      if (br.bad) return TTSB_FLAC_TRUNCATED;
      i += n;
    }
    if (kStore) {
      if (!lpc) {
        for (int t = order; t < block; ++t) {
          int64_t pred = 0;
          if (order == 1) pred = out[t - 1];
          else if (order == 2) pred = 2 * (int64_t)out[t - 1] - out[t - 2];
          else if (order == 3) pred = 3 * (int64_t)out[t - 1] - 3 * (int64_t)out[t - 2] + out[t - 3];
          else if (order == 4) pred = 4 * (int64_t)out[t - 1] - 6 * (int64_t)out[t - 2] + 4 * (int64_t)out[t - 3] - out[t - 4];
          out[t] = (int32_t)(out[t] + pred);
        }
      } else {
        for (int t = order; t < block; ++t) {
          int64_t sum = 0;
          for (int j = 0; j < order; ++j) sum += (int64_t)coef[j * coef_stride] * out[t - 1 - j];
          out[t] = (int32_t)(out[t] + (sum >> shift));
        }
      }
    }
  }
  if (kStore && wasted)
    for (int t = 0; t < block; ++t) out[t] = (int32_t)((uint32_t)out[t] << wasted);
  return 0;
}

__global__ void __launch_bounds__(FLAC_FIND_THREADS)
flac_find_kernel(const uint8_t* __restrict__ data, const FlacFile* __restrict__ files, int32_t* __restrict__ cand_pos,
                 int32_t* __restrict__ cand_count) {
  __shared__ uint8_t crc8[256];
  __shared__ int warp_hits[FLAC_FIND_THREADS / 32];
  flac_tables(crc8, nullptr);
  __syncthreads();
  const FlacFile fd = files[blockIdx.x];
  const uint8_t* f = data + fd.byte_start;
  const int len = fd.byte_len;
  const int blocking = len >= 2 ? (__ldg(f + 1) & 1) : 0;       // the first frame's blocking strategy is the stream's
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int cap = (len + 4) / 5;
  int count = 0;
  for (int base = 0; base < len; base += FLAC_FIND_THREADS) {
    const int pos = base + (int)threadIdx.x;
    FlacHeader h;
    const bool hit = pos < len && __ldg(f + pos) == 0xFF && flac_header(f, len, pos, blocking, fd, crc8, h);
    const unsigned ballot = __ballot_sync(0xffffffffu, hit);
    if (lane == 0) warp_hits[warp] = __popc(ballot);
    __syncthreads();
    int before = 0, all = 0;
#pragma unroll
    for (int w = 0; w < FLAC_FIND_THREADS / 32; ++w) {
      const int s = warp_hits[w];
      before += w < warp ? s : 0;
      all += s;
    }
    const int slot = count + before + __popc(ballot & ((1u << lane) - 1u));
    if (hit && slot < cap) cand_pos[fd.cand_base + slot] = pos;
    count += all;
    __syncthreads();
  }
  if (threadIdx.x == 0) cand_count[blockIdx.x] = min(count, cap);
}

__global__ void __launch_bounds__(FLAC_THREADS, 8)
flac_parse_kernel(const uint8_t* __restrict__ data, const FlacFile* __restrict__ files, const int32_t* __restrict__ cand_pos,
                  const int32_t* __restrict__ cand_count, int32_t* __restrict__ cand_end, int32_t* __restrict__ cand_status) {
  __shared__ uint8_t crc8[256];
  __shared__ uint16_t crc16[256];
  flac_tables(crc8, crc16);
  __syncthreads();
  const FlacFile fd = files[blockIdx.y];
  const uint8_t* f = data + fd.byte_start;
  const int len = fd.byte_len;
  const int blocking = len >= 2 ? (__ldg(f + 1) & 1) : 0;
  const int n = cand_count[blockIdx.y];
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
    const int64_t slot = fd.cand_base + k;
    const int pos = cand_pos[slot];
    FlacHeader h;
    flac_header(f, len, pos, blocking, fd, crc8, h);
    int status = 0, end = pos + h.len;
    if (h.channels != fd.channels || h.bps != fd.bps || h.rate != fd.rate || h.block > fd.max_block) {
      status = TTSB_FLAC_MISMATCH;
    } else {
      FlacBits br;
      br.init(f, len, pos + h.len);
      for (int c = 0; c < h.channels && !status; ++c)
        status = flac_subframe<false>(br, h.block, h.bps + flac_side(h.assign, c), nullptr, nullptr, 0);
      if (!status) {
        const int pad = (int)(br.tell() & 7);
        if (pad && br.get(8 - pad) != 0) status = br.bad ? TTSB_FLAC_TRUNCATED : TTSB_FLAC_BAD_FRAME;
      }
      if (!status) {
        const uint32_t want = br.get(16);
        if (br.bad) {
          status = TTSB_FLAC_TRUNCATED;
        } else {
          end = (int)(br.tell() >> 3);
          uint32_t crc = 0;
          for (int b = pos; b < end - 2; ++b) crc = ((crc << 8) & 0xFFFFu) ^ crc16[(crc >> 8) ^ __ldg(f + b)];
          if (crc != want) status = TTSB_FLAC_CRC;
        }
      }
    }
    cand_end[slot] = end;
    cand_status[slot] = status;
  }
}

__global__ void flac_chain_kernel(const uint8_t* __restrict__ data, const FlacFile* __restrict__ files, int n_files,
                                  const int32_t* __restrict__ cand_pos, const int32_t* __restrict__ cand_count,
                                  const int32_t* __restrict__ cand_end, const int32_t* __restrict__ cand_status,
                                  FlacFrame* __restrict__ frames, int32_t* __restrict__ frame_count, int32_t* __restrict__ status_out) {
  __shared__ uint8_t crc8[256];
  flac_tables(crc8, nullptr);
  __syncthreads();
  for (int fi = blockIdx.x * blockDim.x + threadIdx.x; fi < n_files; fi += gridDim.x * blockDim.x) {
    const FlacFile fd = files[fi];
    const uint8_t* f = data + fd.byte_start;
    const int32_t* cands = cand_pos + fd.cand_base;
    const int n = cand_count[fi];
    const int blocking = fd.byte_len >= 2 ? (__ldg(f + 1) & 1) : 0;
    int status = 0, idx = 0, pos = 0, first_block = 0;
    int64_t decoded = 0;
    while (decoded < fd.total) {
      if (pos >= fd.byte_len) { status = TTSB_FLAC_TRUNCATED; break; }
      int lo = 0, hi = n;                          // the first candidate at or after pos
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (cands[mid] < pos) lo = mid + 1; else hi = mid;
      }
      if (lo == n || cands[lo] != pos) { status = TTSB_FLAC_NO_SYNC; break; }
      const int64_t slot = fd.cand_base + lo;
      if (cand_status[slot]) { status = cand_status[slot]; break; }
      FlacHeader h;
      flac_header(f, fd.byte_len, pos, blocking, fd, crc8, h);
      if (decoded + h.block > fd.total) { status = TTSB_FLAC_TOTAL; break; }
      const bool last = decoded + h.block == fd.total;
      if (idx == 0) first_block = h.block;
      if (!last && (h.block < fd.min_block || (!blocking && h.block != first_block))) { status = TTSB_FLAC_MISMATCH; break; }
      if (h.number != (blocking ? decoded : (int64_t)idx)) { status = TTSB_FLAC_NUMBER; break; }
      if (idx >= fd.frame_cap) { status = TTSB_FLAC_MISMATCH; break; }
      frames[fd.frame_base + idx] = FlacFrame{decoded, pos, h.block, h.assign, 0};
      ++idx;
      decoded += h.block;
      pos = cand_end[slot];
    }
    frame_count[fi] = status ? 0 : idx;
    status_out[2 * fi] = status;
    status_out[2 * fi + 1] = idx;
  }
}

__global__ void __launch_bounds__(FLAC_THREADS, 8)
flac_decode_kernel(const uint8_t* __restrict__ data, const FlacFile* __restrict__ files, const FlacFrame* __restrict__ frames,
                   const int32_t* __restrict__ frame_count, int32_t* __restrict__ planes) {
  __shared__ int32_t coef[FLAC_MAX_LPC * FLAC_THREADS];          // thread t's coefficient j at j * FLAC_THREADS + t
  const FlacFile fd = files[blockIdx.y];
  const uint8_t* f = data + fd.byte_start;
  const int C = fd.channels;
  const int n = frame_count[blockIdx.y] * C;
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
    const FlacFrame fr = frames[fd.frame_base + k / C];
    const int c = k % C;
    FlacBits br;
    br.init(f, fd.byte_len, fr.pos + flac_header_len(f + fr.pos));
    for (int j = 0; j < c; ++j) flac_subframe<false>(br, fr.block, fd.bps + flac_side(fr.assign, j), nullptr, nullptr, 0);
    flac_subframe<true>(br, fr.block, fd.bps + flac_side(fr.assign, c), planes + fd.plane_base + c * fd.total + fr.start,
                        coef + threadIdx.x, FLAC_THREADS);
  }
}

__device__ __forceinline__ int flac_find_file(const FlacFile* __restrict__ files, int n, int64_t g) {
  int lo = 0, hi = n;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (files[mid].mono_base <= g) lo = mid; else hi = mid;
  }
  return lo;
}

__global__ void flac_output_kernel(const FlacFile* __restrict__ files, int n_files, int64_t total, const FlacFrame* __restrict__ frames,
                                   const int32_t* __restrict__ frame_count, const int32_t* __restrict__ planes,
                                   const int32_t* __restrict__ status, float* __restrict__ mono_out, int32_t* __restrict__ pcm_out) {
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (int64_t)gridDim.x * blockDim.x) {
    const int fi = flac_find_file(files, n_files, g);
    const FlacFile fd = files[fi];
    const int64_t i = g - fd.mono_base;
    const int C = fd.channels;
    int32_t v[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) v[c] = 0;
    if (status[2 * fi] == 0) {
#pragma unroll
      for (int c = 0; c < 8; ++c)
        if (c < C) v[c] = planes[fd.plane_base + c * fd.total + i];
      if (C == 2) {
        const FlacFrame* fr = frames + fd.frame_base;   // the frame holding sample i
        int lo = 0, hi = frame_count[fi];
        while (hi - lo > 1) {
          const int mid = (lo + hi) >> 1;
          if (fr[mid].start <= i) lo = mid; else hi = mid;
        }
        const int assign = fr[lo].assign;
        if (assign == 8) v[1] = v[0] - v[1];
        else if (assign == 9) v[0] = v[0] + v[1];
        else if (assign == 10) {
          const int32_t mid = (int32_t)((uint32_t)v[0] << 1) | (v[1] & 1), side = v[1];
          v[0] = (mid + side) >> 1;
          v[1] = (mid - side) >> 1;
        }
      }
    }
    const float scale = __int_as_float((128 - fd.bps) << 23);     // 2^-(bps - 1)
    float x[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) x[c] = __fmul_rn((float)v[c], scale);
    float m;
    if (C == 8) {
      m = __fadd_rn(__fadd_rn(__fadd_rn(x[0], x[1]), __fadd_rn(x[2], x[3])), __fadd_rn(__fadd_rn(x[4], x[5]), __fadd_rn(x[6], x[7])));
    } else {
      m = x[0];
#pragma unroll
      for (int c = 1; c < 7; ++c)
        if (c < C) m = __fadd_rn(m, x[c]);
    }
    mono_out[g] = C == 1 ? m : __fdiv_rn(m, (float)C);
    if (pcm_out) {
#pragma unroll
      for (int c = 0; c < 8; ++c)
        if (c < C) pcm_out[fd.pcm_base + i * C + c] = v[c];
    }
  }
}

int flac_bad(const char* fmt, long long a = 0, long long b = 0) {
  set_last_error(fmt, a, b);
  return TTSB_ERR_INVALID_ARGUMENT;
}

size_t flac_align16(size_t x) { return (x + 15) & ~(size_t)15; }

struct FlacPlan {
  std::vector<FlacFile> files;
  int64_t cand_slots = 0, frame_slots = 0, plane_values = 0, mono = 0, pcm = 0;
  int max_frames = 1, max_units = 1;
  size_t off_cand = 0, off_count = 0, off_end = 0, off_status = 0, off_frames = 0, off_fcount = 0, off_planes = 0;
  int64_t bytes = 0;
};

// Checks the host tables and lays out the workspace: file table, candidate positions / counts / ends / statuses, frame table,
// frame counts, planar PCM.
int flac_plan(const int64_t* byte_offsets, const int64_t* info, int n_files, FlacPlan& p) {
  if (!byte_offsets || !info) return flac_bad("ttsb_flac_decode: NULL byte_offsets or stream info");
  if (n_files < 1 || n_files > 65535) return flac_bad("ttsb_flac_decode: n_files %lld outside [1, 65535]", n_files);
  if (byte_offsets[0] != 0) return flac_bad("ttsb_flac_decode: byte_offsets must start at 0, got %lld", byte_offsets[0]);
  p.files.resize(n_files);
  for (int i = 0; i < n_files; ++i) {
    const int64_t* si = info + (size_t)i * TTSB_FLAC_INFO_FIELDS;
    const long long channels = si[0], bps = si[1], rate = si[2], min_block = si[3], max_block = si[4], total = si[5];
    const long long len = byte_offsets[i + 1] - byte_offsets[i];
    if (len < 0) return flac_bad("ttsb_flac_decode: byte_offsets decrease at file %lld", i);
    if (len > INT32_MAX) return flac_bad("ttsb_flac_decode: file %lld has %lld frame bytes (at most 2^31 - 1)", i, len);
    if (channels < 1 || channels > 8) return flac_bad("ttsb_flac_decode: file %lld has %lld channels (1 to 8)", i, channels);
    if (bps > 24 && bps <= 32)
      return flac_bad("ttsb_flac_decode: file %lld is %lld-bit; 25- to 32-bit FLAC is not supported", i, bps);
    if (bps < 4 || bps > 24)
      return flac_bad("ttsb_flac_decode: file %lld has %lld bits per sample (4 to 24)", i, bps);
    if (rate < 1 || rate > 1048575) return flac_bad("ttsb_flac_decode: file %lld has sample rate %lld", i, rate);
    if (max_block > 65535) return flac_bad("ttsb_flac_decode: file %lld has max block size %lld (at most 65535)", i, max_block);
    if (min_block < 16 || min_block > max_block)
      return flac_bad("ttsb_flac_decode: file %lld has min block size %lld (16 to the max block size)", i, min_block);
    if (total < 1 || total > ((int64_t)1 << 36))
      return flac_bad("ttsb_flac_decode: file %lld has total_samples %lld (must be known and positive)", i, total);
    FlacFile& fd = p.files[i];
    fd.byte_start = byte_offsets[i];
    fd.byte_len = (int32_t)len;
    fd.total = total;
    fd.channels = (int32_t)channels;
    fd.bps = (int32_t)bps;
    fd.rate = (int32_t)rate;
    fd.min_block = (int32_t)min_block;
    fd.max_block = (int32_t)max_block;
    const int64_t frames = (total + min_block - 1) / min_block + 1;
    if (frames > INT32_MAX) return flac_bad("ttsb_flac_decode: file %lld has too many frames", i);
    fd.frame_cap = (int32_t)frames;
    fd.cand_base = p.cand_slots;
    fd.frame_base = p.frame_slots;
    fd.plane_base = p.plane_values;
    fd.mono_base = p.mono;
    fd.pcm_base = p.pcm;
    p.cand_slots += (len + 4) / 5;
    p.frame_slots += frames;
    p.plane_values += total * channels;
    p.mono += total;
    p.pcm += total * channels;
    p.max_frames = (int)std::min<int64_t>(std::max<int64_t>(p.max_frames, frames), INT32_MAX);
    p.max_units = (int)std::min<int64_t>(std::max<int64_t>(p.max_units, frames * channels), INT32_MAX);
  }
  size_t off = flac_align16((size_t)n_files * sizeof(FlacFile));
  p.off_cand = off;
  off = flac_align16(off + (size_t)p.cand_slots * sizeof(int32_t));
  p.off_count = off;
  off = flac_align16(off + (size_t)n_files * sizeof(int32_t));
  p.off_end = off;
  off = flac_align16(off + (size_t)p.cand_slots * sizeof(int32_t));
  p.off_status = off;
  off = flac_align16(off + (size_t)p.cand_slots * sizeof(int32_t));
  p.off_frames = off;
  off = flac_align16(off + (size_t)p.frame_slots * sizeof(FlacFrame));
  p.off_fcount = off;
  off = flac_align16(off + (size_t)n_files * sizeof(int32_t));
  p.off_planes = off;
  p.bytes = (int64_t)(off + (size_t)p.plane_values * sizeof(int32_t));
  return 0;
}

}  // namespace
}  // namespace ttsb

using namespace ttsb;

extern "C" int64_t ttsb_flac_decode_workspace_bytes(const int64_t* byte_offsets, const int64_t* info, int n_files) {
  FlacPlan p;
  if (flac_plan(byte_offsets, info, n_files, p)) return -1;
  return p.bytes;
}

extern "C" int ttsb_flac_decode_batch(const uint8_t* data, const int64_t* byte_offsets, const int64_t* info, int n_files,
                                      float* mono_out, int32_t* pcm_out, int32_t* status_out, void* workspace,
                                      int64_t workspace_bytes, void* stream_v) {
  if (!workspace || !mono_out || !status_out) return flac_bad("ttsb_flac_decode: NULL pointer");
  FlacPlan p;
  int rc = flac_plan(byte_offsets, info, n_files, p);
  if (rc) return rc;
  if (!data && byte_offsets[n_files] > 0) return flac_bad("ttsb_flac_decode: NULL data");
  if (workspace_bytes < p.bytes) return flac_bad("ttsb_flac_decode: workspace too small (%lld bytes, need %lld)", workspace_bytes, p.bytes);
  if (reinterpret_cast<uintptr_t>(workspace) % 16 != 0) return flac_bad("ttsb_flac_decode: workspace must be 16-byte aligned");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  TTSB_CUDA_OK(cudaMemcpyAsync(ws, p.files.data(), p.files.size() * sizeof(FlacFile), cudaMemcpyHostToDevice, stream));
  const FlacFile* files = reinterpret_cast<const FlacFile*>(ws);
  int32_t* cand = reinterpret_cast<int32_t*>(ws + p.off_cand);
  int32_t* count = reinterpret_cast<int32_t*>(ws + p.off_count);
  int32_t* cend = reinterpret_cast<int32_t*>(ws + p.off_end);
  int32_t* cstatus = reinterpret_cast<int32_t*>(ws + p.off_status);
  FlacFrame* frames = reinterpret_cast<FlacFrame*>(ws + p.off_frames);
  int32_t* fcount = reinterpret_cast<int32_t*>(ws + p.off_fcount);
  int32_t* planes = reinterpret_cast<int32_t*>(ws + p.off_planes);

  flac_find_kernel<<<n_files, FLAC_FIND_THREADS, 0, stream>>>(data, files, cand, count);
  count_launch();
  rc = check_cuda(cudaGetLastError(), "flac_find_kernel launch");
  if (rc) return rc;
  const dim3 parse_grid((unsigned)std::min(((int64_t)p.max_frames + FLAC_THREADS - 1) / FLAC_THREADS, (int64_t)1024), (unsigned)n_files);
  flac_parse_kernel<<<parse_grid, FLAC_THREADS, 0, stream>>>(data, files, cand, count, cend, cstatus);
  count_launch();
  rc = check_cuda(cudaGetLastError(), "flac_parse_kernel launch");
  if (rc) return rc;
  flac_chain_kernel<<<(n_files + FLAC_THREADS - 1) / FLAC_THREADS, FLAC_THREADS, 0, stream>>>(data, files, n_files, cand, count, cend,
                                                                                              cstatus, frames, fcount, status_out);
  count_launch();
  rc = check_cuda(cudaGetLastError(), "flac_chain_kernel launch");
  if (rc) return rc;
  const dim3 decode_grid((unsigned)std::min(((int64_t)p.max_units + FLAC_THREADS - 1) / FLAC_THREADS, (int64_t)1024), (unsigned)n_files);
  flac_decode_kernel<<<decode_grid, FLAC_THREADS, 0, stream>>>(data, files, frames, fcount, planes);
  count_launch();
  rc = check_cuda(cudaGetLastError(), "flac_decode_kernel launch");
  if (rc) return rc;
  const int grid = (int)std::min((p.mono + 255) / 256, (int64_t)16 * num_sms());
  flac_output_kernel<<<grid, 256, 0, stream>>>(files, n_files, p.mono, frames, fcount, planes, status_out, mono_out, pcm_out);
  count_launch();
  return check_cuda(cudaGetLastError(), "flac_output_kernel launch");
}
