// Decoding of one 8-bit grayscale PNG image stream (zlib / deflate, RFC 1950 / 1951, then the PNG row filters) into an (h, w)
// uint8 plane, as libpng under cv2.imdecode(..., IMREAD_GRAYSCALE) decodes it (lav/utils/datasets/basic_dataset.py:94,99).
//
// Written once for the device and the host: on the device one warp decodes one image (all 32 lanes run the symbol decode
// redundantly, so every lane holds the same state without a broadcast, and they split the byte copies, the Adler-32 sum and the
// None / Up / Sub rows); on the host the same functions run with one lane, which lets the decoder be checked against zlib and
// cv2 without a GPU.  Every read is bounded by the stream's length and every write by the plane: a malformed stream returns a
// nonzero PngStatus and writes nothing outside its own plane.
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define LAVB_HD __host__ __device__ __forceinline__
#else
#define LAVB_HD inline
#endif

namespace lavb_png {

enum PngStatus : int {
  kOk = 0,
  kBadJob = 1,         // job outside the source buffer or the output planes, or of another size than the launch's planes
  kBadHeader = 2,      // zlib header: CM != 8, CINFO > 7, FCHECK, or a preset dictionary
  kTruncated = 3,      // the stream ends before the final block and the Adler-32 trailer
  kBadBlockType = 4,   // BTYPE 3
  kBadStored = 5,      // stored block LEN != ~NLEN
  kBadCodeLengths = 6, // oversubscribed / incomplete code, too many symbols, bad repeat, no end-of-block code
  kBadSymbol = 7,      // a code with no symbol, length symbol 286/287, distance code 30/31
  kBadDistance = 8,    // a match reaching before the start of the output
  kBadSize = 9,        // the inflated size is not h * (w + 1)
  kBadAdler = 10,      // Adler-32 of the inflated bytes differs from the trailer
  kBadFilter = 11,     // a row filter byte > 4
};

constexpr int kFastBits = 10;

// a canonical Huffman code: a 2^kFastBits lookup of codes up to kFastBits long ((symbol << 4) | length, 0 = longer or none),
// and the counts / length-sorted symbols of the bit-by-bit decode of the longer codes
struct Huff {
  uint16_t fast[1 << kFastBits];
  uint16_t count[16];
  uint16_t sym[288];
};

struct Scratch {                 // per image: shared memory on the device
  Huff lit, dist;                // `dist` also holds the code-length code while a dynamic header is read
  uint8_t lens[288 + 32];
};

// the lanes of a warp on the device, one lane on the host
struct Lanes {
  int lane, n;
  LAVB_HD void sync() const {
#ifdef __CUDA_ARCH__
    __syncwarp();
#endif
  }
  LAVB_HD unsigned long long sum(unsigned long long v) const {
#ifdef __CUDA_ARCH__
    for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
#endif
    return v;
  }
};

// the inflated stream is h rows of (filter byte, w pixels): pixels go straight to the plane, filter bytes to `filt`
struct Sink {
  uint8_t* plane;
  uint8_t* filt;
  int w1;                        // w + 1
  LAVB_HD void put(int p, uint8_t v) const {
    const int r = p / w1, c = p - r * w1;
    if (c == 0) filt[r] = v;
    else plane[r * (w1 - 1) + c - 1] = v;
  }
  LAVB_HD uint8_t get(int p) const {
    const int r = p / w1, c = p - r * w1;
    return c == 0 ? filt[r] : plane[r * (w1 - 1) + c - 1];
  }
};

// LSB-first bit reader; reads past the end yield zeros and are caught by overrun()
struct Bits {
  const uint8_t* src;
  long long len, in;
  unsigned long long buf;
  int cnt;
  LAVB_HD void refill() {
    while (cnt <= 56) {
      const unsigned long long b = in < len ? src[in] : 0;
      buf |= b << cnt;
      ++in;
      cnt += 8;
    }
  }
  LAVB_HD unsigned peek(int n) { refill(); return (unsigned)(buf & ((1ull << n) - 1)); }
  LAVB_HD void drop(int n) { buf >>= n; cnt -= n; }
  LAVB_HD unsigned get(int n) {
    if (n == 0) return 0;
    const unsigned v = peek(n);
    drop(n);
    return v;
  }
  LAVB_HD bool overrun() const { return in * 8 - cnt > len * 8; }
  LAVB_HD void align() { drop(cnt & 7); }
};

LAVB_HD unsigned reverse_bits(unsigned v, int n) {
  unsigned r = 0;
  for (int i = 0; i < n; ++i) r = (r << 1) | ((v >> i) & 1);
  return r;
}

// builds h from the code lengths lens[0..n); the rules of zlib's inflate_table: an oversubscribed set is an error, and an
// incomplete one too, except for a literal / distance code whose only code is one bit long (codes = false)
LAVB_HD int build(Huff& h, const uint8_t* lens, int n, bool codes, const Lanes& L) {
  int count[16] = {0};
  for (int s = 0; s < n; ++s) ++count[lens[s]];
  int left = 1, max = 0;
  for (int l = 1; l < 16; ++l) {
    left = (left << 1) - count[l];
    if (left < 0) return kBadCodeLengths;
    if (count[l]) max = l;
  }
  if (max > 0 && left > 0 && (codes || max != 1)) return kBadCodeLengths;
  int offs[16], first[16];
  offs[1] = 0;
  for (int l = 1; l < 15; ++l) offs[l + 1] = offs[l] + count[l];
  int code = 0;
  for (int l = 1; l < 16; ++l) {
    first[l] = code;
    code = (code + count[l]) << 1;
  }
  L.sync();                                         // every lane is done reading the previous code held in h
  for (int i = L.lane; i < (1 << kFastBits); i += L.n) h.fast[i] = 0;
  for (int l = L.lane; l < 16; l += L.n) h.count[l] = (uint16_t)(l ? count[l] : 0);
  if (L.lane == 0) {
    int o[16];
    for (int l = 0; l < 16; ++l) o[l] = offs[l];
    for (int s = 0; s < n; ++s)
      if (lens[s]) h.sym[o[lens[s]]++] = (uint16_t)s;
  }
  L.sync();
  const int total = offs[15] + count[15];
  for (int i = L.lane; i < total; i += L.n) {
    const int s = h.sym[i], l = lens[s];
    if (l > kFastBits) continue;
    const unsigned r = reverse_bits((unsigned)(first[l] + i - offs[l]), l);
    for (unsigned e = r; e < (1u << kFastBits); e += 1u << l) h.fast[e] = (uint16_t)((s << 4) | l);
  }
  L.sync();
  return kOk;
}

// the next symbol of code h, or -1 for a bit sequence that is no code
LAVB_HD int decode(const Huff& h, Bits& b) {
  const unsigned v = b.peek(15);
  const unsigned e = h.fast[v & ((1u << kFastBits) - 1)];
  if (e) {
    b.drop(e & 15);
    return (int)(e >> 4);
  }
  int code = 0, first = 0, index = 0;
  for (int l = 1; l < 16; ++l) {
    code |= (v >> (l - 1)) & 1;
    const int count = h.count[l];
    if (code - count < first) {
      b.drop(l);
      return h.sym[index + (code - first)];
    }
    index += count;
    first = (first + count) << 1;
    code <<= 1;
  }
  return -1;
}

// length symbol 257 + i: base 3..258 and extra bits; distance symbol i: base 1..24577 and extra bits (RFC 1951 3.2.5)
LAVB_HD int len_extra(int i) { return i < 8 || i == 28 ? 0 : (i - 4) >> 2; }
LAVB_HD int len_base(int i) { return i < 8 ? 3 + i : i == 28 ? 258 : ((4 + (i & 3)) << len_extra(i)) + 3; }
LAVB_HD int dist_extra(int i) { return i < 4 ? 0 : (i >> 1) - 1; }
LAVB_HD int dist_base(int i) { return i < 4 ? 1 + i : ((2 + (i & 1)) << dist_extra(i)) + 1; }

LAVB_HD int dynamic_header(Scratch& s, Bits& b, const Lanes& L) {
  const int nlen = (int)b.get(5) + 257, ndist = (int)b.get(5) + 1, ncode = (int)b.get(4) + 4;
  if (nlen > 286 || ndist > 30) return kBadCodeLengths;
  const char* order = "\x10\x11\x12\x00\x08\x07\x09\x06\x0a\x05\x0b\x04\x0c\x03\x0d\x02\x0e\x01\x0f";
  uint8_t cl[19];
  for (int i = 0; i < 19; ++i) cl[i] = 0;
  for (int i = 0; i < ncode; ++i) cl[(int)order[i]] = (uint8_t)b.get(3);
  int st = build(s.dist, cl, 19, true, L);
  if (st) return st;
  int i = 0, prev = -1;
  while (i < nlen + ndist) {
    const int sym = decode(s.dist, b);
    if (sym < 0) return kBadCodeLengths;
    if (sym < 16) {
      if (L.lane == 0) s.lens[i] = (uint8_t)sym;
      prev = sym;
      ++i;
      continue;
    }
    int len = 0, rep;
    if (sym == 16) {
      if (prev < 0) return kBadCodeLengths;
      len = prev;
      rep = 3 + (int)b.get(2);
    } else if (sym == 17) {
      rep = 3 + (int)b.get(3);
    } else {
      rep = 11 + (int)b.get(7);
    }
    if (i + rep > nlen + ndist) return kBadCodeLengths;
    if (L.lane == 0)
      for (int k = 0; k < rep; ++k) s.lens[i + k] = (uint8_t)len;
    prev = len;
    i += rep;
  }
  if (b.overrun()) return kTruncated;
  L.sync();
  if (s.lens[256] == 0) return kBadCodeLengths;
  if ((st = build(s.lit, s.lens, nlen, false, L))) return st;
  return build(s.dist, s.lens + nlen, ndist, false, L);
}

LAVB_HD int fixed_tables(Scratch& s, const Lanes& L) {
  L.sync();
  for (int i = L.lane; i < 288 + 32; i += L.n) s.lens[i] = (uint8_t)(i < 144 ? 8 : i < 256 ? 9 : i < 280 ? 7 : i < 288 ? 8 : 5);
  L.sync();
  const int st = build(s.lit, s.lens, 288, false, L);
  return st ? st : build(s.dist, s.lens + 288, 32, false, L);
}

// the Huffman-coded data of one block; *out = inflated bytes so far
LAVB_HD int codes(const Scratch& s, Bits& b, const Sink& o, int n_out, int* out, const Lanes& L) {
  int pos = *out;
  for (;;) {
    const int sym = decode(s.lit, b);
    if (b.overrun()) return kTruncated;
    if (sym < 0) return kBadSymbol;
    if (sym < 256) {
      if (pos >= n_out) return kBadSize;
      if (L.lane == 0) o.put(pos, (uint8_t)sym);
      ++pos;
      continue;
    }
    if (sym == 256) break;
    const int li = sym - 257;
    if (li >= 29) return kBadSymbol;
    const int len = len_base(li) + (int)b.get(len_extra(li));
    const int ds = decode(s.dist, b);
    if (ds < 0 || ds >= 30) return kBadSymbol;
    const int dist = dist_base(ds) + (int)b.get(dist_extra(ds));
    if (b.overrun()) return kTruncated;
    if (dist > pos) return kBadDistance;
    if (len > n_out - pos) return kBadSize;
    L.sync();                                       // the bytes this match reads were written by any lane
    // out[pos + k] = out[pos - dist + k], k in order, equals out[pos - dist + k % dist]: every source byte precedes pos
    for (int k = L.lane; k < len; k += L.n) o.put(pos + k, o.get(pos - dist + (dist >= len ? k : k % dist)));
    pos += len;
  }
  *out = pos;
  return kOk;
}

// the zlib stream src[0..len) -> filtered rows (pixels in plane, filter bytes in filt); then the Adler-32 check
LAVB_HD int inflate(Scratch& s, const uint8_t* src, long long len, const Sink& o, int n_out, const Lanes& L) {
  Bits b{src, len, 0, 0, 0};
  const unsigned cmf = b.get(8), flg = b.get(8);
  if (b.overrun() || (cmf & 15) != 8 || (cmf >> 4) > 7 || (cmf * 256 + flg) % 31 != 0 || (flg & 0x20)) return kBadHeader;
  int pos = 0, last = 0;
  while (!last) {
    last = (int)b.get(1);
    const int type = (int)b.get(2);
    int st;
    if (type == 0) {
      b.align();
      const unsigned n = b.get(16), nn = b.get(16);
      if (b.overrun()) return kTruncated;
      if (n != (~nn & 0xffffu)) return kBadStored;
      const long long at = b.in - b.cnt / 8;        // the buffered bytes are whole bytes after align()
      if (at + n > len) return kTruncated;
      if ((int)n > n_out - pos) return kBadSize;
      L.sync();
      for (int k = L.lane; k < (int)n; k += L.n) o.put(pos + k, src[at + k]);
      pos += (int)n;
      b.in = at + n;
      b.buf = 0;
      b.cnt = 0;
      continue;
    }
    if (type == 1) st = fixed_tables(s, L);
    else if (type == 2) st = dynamic_header(s, b, L);
    else return kBadBlockType;
    if (st) return st;
    if ((st = codes(s, b, o, n_out, &pos, L))) return st;
  }
  if (pos != n_out) return kBadSize;
  b.align();
  unsigned want = 0;
  for (int k = 0; k < 4; ++k) want = (want << 8) | b.get(8);
  if (b.overrun()) return kTruncated;
  // Adler-32: A = 1 + sum x_k, B = n + sum (n - k) x_k (k = 0 .. n-1), both mod 65521
  L.sync();
  unsigned long long a = 0, bb = 0;
  for (int p = L.lane; p < n_out; p += L.n) {
    const unsigned x = o.get(p);
    a += x;
    bb += (unsigned long long)(n_out - p) * x;
  }
  a = L.sum(a);
  bb = L.sum(bb);
  const unsigned got = (unsigned)(((bb + (unsigned long long)n_out) % 65521ull) << 16) | (unsigned)((a + 1) % 65521ull);
  return got == want ? kOk : kBadAdler;
}

LAVB_HD int paeth(int a, int b, int c) {
  const int p = a + b - c, pa = p > a ? p - a : a - p, pb = p > b ? p - b : b - p, pc = p > c ? p - c : c - p;
  return (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c);
}

// undoes the row filters in place, top to bottom (bpp = 1)
LAVB_HD int unfilter(uint8_t* plane, const uint8_t* filt, int h, int w, const Lanes& L) {
  for (int r = 0; r < h; ++r)
    if (filt[r] > 4) return kBadFilter;
  for (int r = 0; r < h; ++r) {
    uint8_t* cur = plane + (long long)r * w;
    const uint8_t* prv = cur - w;
    switch (filt[r]) {
      case 1: {                                     // Sub: an inclusive prefix sum mod 256 along the row
#ifdef __CUDA_ARCH__
        int carry = 0;
        for (int c0 = 0; c0 < w; c0 += 32) {
          const int c = c0 + L.lane;
          int v = c < w ? cur[c] : 0;
          for (int d = 1; d < 32; d <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, v, d);
            if (L.lane >= d) v += t;
          }
          v += carry;
          if (c < w) cur[c] = (uint8_t)v;
          carry = __shfl_sync(0xffffffffu, v, 31) & 255;
        }
#else
        for (int c = 1; c < w; ++c) cur[c] = (uint8_t)(cur[c] + cur[c - 1]);
#endif
        break;
      }
      case 2:
        if (r > 0)
          for (int c = L.lane; c < w; c += L.n) cur[c] = (uint8_t)(cur[c] + prv[c]);
        break;
      case 3:
        if (L.lane == 0)
          for (int c = 0; c < w; ++c) cur[c] = (uint8_t)(cur[c] + (((c ? cur[c - 1] : 0) + (r ? prv[c] : 0)) >> 1));
        break;
      case 4:
        if (L.lane == 0)
          for (int c = 0; c < w; ++c)
            cur[c] = (uint8_t)(cur[c] + paeth(c ? cur[c - 1] : 0, r ? prv[c] : 0, (r && c) ? prv[c - 1] : 0));
        break;
      default:
        break;
    }
    L.sync();
  }
  return kOk;
}

// one image: the zlib stream src[0..len) -> the (h, w) plane; filt = h bytes of scratch
LAVB_HD int decode_gray8(Scratch& s, uint8_t* filt, const uint8_t* src, long long len, uint8_t* plane, int h, int w,
                         const Lanes& L) {
  const Sink o{plane, filt, w + 1};
  const int st = inflate(s, src, len, o, h * (w + 1), L);
  L.sync();
  return st ? st : unfilter(plane, filt, h, w, L);
}

}  // namespace lavb_png
