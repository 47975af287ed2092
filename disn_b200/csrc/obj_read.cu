// OBJ file -> the resident mesh, parsed on the device.  The specification is create_sdf.read_obj / read_obj_parts: every
// file inside the grammar below gives their arrays bit for bit; every other file is refused with DISN_ERR_OBJ_UNSUPPORTED
// (the caller's fallback is the Python reader, so behaviour outside the grammar is the Python reader's by construction).
//
// Grammar (what Python does with the text): ASCII bytes only; lines end at "\n", "\r\n" or a lone "\r" (universal
// newlines); tokens are separated by the ASCII characters str.split() splits on (space, \t, \v, \f, \x1c-\x1f); the first
// token selects the record: `v` (tokens 1-3 are coordinates), `f` (exactly three corners) or `usemtl` (parts), anything
// else is ignored.  A coordinate is [+-]?(digits[.digits?]|.digits)([eE][+-]?digits)? or inf / infinity / nan in any case
// with an optional sign; its value is the correctly rounded float64, then rounded to float32.  A corner is the text
// before its first '/': [+-]?digits with at most 18 digits and a value in [1, V], V the `v` records of the whole file.
//
// Phases on the context's stream: upload -> line starts (a byte pass counts them and flags non-ASCII bytes, then a device
// select compacts them) -> classification (one thread per line reads its first token) and an inclusive scan of the
// (v, f) counts -> parse (one thread per v / f line writes straight into the resident mesh).  A coordinate is computed on
// the device when its significand has <= 19 significant digits, is <= 2^53 and the decimal exponent is within +-22: one
// IEEE multiply or divide by an exact power of ten, then one rounding to float32.  Every other valid coordinate goes on
// a list that the host converts with std::from_chars<double> and patches into the vertices.
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>

#include <algorithm>
#include <charconv>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <map>
#include <string>

#include "common.cuh"

namespace disn {
namespace {

enum : uint8_t { REC_OTHER = 0, REC_V = 1, REC_F = 2, REC_MTL = 3 };
// reasons a file is refused; the status word is (line << 8) | reason, minimised over the file
enum : uint32_t { BAD_NONE = 0, BAD_COORD = 1, BAD_FEW_COORDS = 2, BAD_CORNERS = 3, BAD_INDEX = 4 };
const char* const kReason[] = {"", "coordinate outside the reader's grammar", "fewer than 3 coordinates",
                               "only triangle faces are supported", "face index outside the reader's grammar or [1, V]"};
constexpr unsigned long long kNoStatus = ~0ull;
constexpr int OBJ_THREADS = 256;

__constant__ double kPow10[23] = {1e0,  1e1,  1e2,  1e3,  1e4,  1e5,  1e6,  1e7,  1e8,  1e9,  1e10, 1e11,
                                  1e12, 1e13, 1e14, 1e15, 1e16, 1e17, 1e18, 1e19, 1e20, 1e21, 1e22};

__host__ __device__ __forceinline__ bool is_sep(uint8_t ch) {      // str.split()'s ASCII whitespace within a line
  return ch == ' ' || ch == '\t' || ch == '\v' || ch == '\f' || (ch >= 0x1c && ch <= 0x1f);
}
__host__ __device__ __forceinline__ bool is_eol(uint8_t ch) { return ch == '\n' || ch == '\r'; }
__host__ __device__ __forceinline__ bool is_digit(uint8_t ch) { return ch >= '0' && ch <= '9'; }
__host__ __device__ __forceinline__ uint8_t lower(uint8_t ch) { return (ch >= 'A' && ch <= 'Z') ? ch + 32 : ch; }

// byte i starts a line: the first byte, or the byte after a line end ("\n", or "\r" not followed by "\n")
__host__ __device__ __forceinline__ bool line_starts_at(const uint8_t* b, int64_t n, int64_t i) {
  if (i == 0) return true;
  const uint8_t p = b[i - 1];
  return p == '\n' || (p == '\r' && b[i] != '\n');
}

struct IsLineStart {
  const uint8_t* b;
  int64_t n;
  __device__ bool operator()(long long i) const { return line_starts_at(b, n, i); }
};

struct MaxOp {
  __device__ int32_t operator()(int32_t a, int32_t b) const { return a > b ? a : b; }
};

// next token of a line from p: [*tb, *te); false at the line's end
__host__ __device__ __forceinline__ bool next_token(const uint8_t*& p, const uint8_t* end, const uint8_t** tb,
                                                    const uint8_t** te) {
  while (p < end && is_sep(*p)) ++p;
  if (p >= end || is_eol(*p)) return false;
  *tb = p;
  while (p < end && !is_sep(*p) && !is_eol(*p)) ++p;
  *te = p;
  return true;
}

// inf / infinity / nan in any case (after the sign)
__host__ __device__ __forceinline__ bool is_special_word(const uint8_t* s, int64_t len) {
  const char* words[3] = {"inf", "infinity", "nan"};
  for (const char* w : words) {
    int64_t k = 0;
    while (w[k] && k < len && lower(s[k]) == (uint8_t)w[k]) ++k;
    if (!w[k] && k == len) return true;
  }
  return false;
}

// Decimal coordinate token [s, e): -1 outside the grammar; 1 when the fast rule applies (value in *out); 0 when it is
// valid but left to the host.  *neg: its sign; *m, *e10: the significand without leading zeros and its decimal exponent.
struct Decimal {
  bool neg;
  uint64_t m;
  int nd;          // significant digits (after leading zeros)
  long long e10;   // value = m * 10^e10 when nd <= 19
};

__host__ __device__ __forceinline__ int scan_decimal(const uint8_t* s, const uint8_t* e, Decimal* d) {
  d->neg = false; d->m = 0; d->nd = 0; d->e10 = 0;
  if (s < e && (*s == '+' || *s == '-')) { d->neg = *s == '-'; ++s; }
  if (s < e && !is_digit(*s) && *s != '.') return is_special_word(s, e - s) ? 0 : -1;
  int n_int = 0, n_frac = 0;
  long long frac = 0;
  for (; s < e && is_digit(*s); ++s, ++n_int) {
    const int dg = *s - '0';
    if (d->nd || dg) { if (d->nd < 19) d->m = d->m * 10 + dg; else ++frac; ++d->nd; }
  }
  if (s < e && *s == '.') {
    ++s;
    for (; s < e && is_digit(*s); ++s, ++n_frac) {
      const int dg = *s - '0';
      if (d->nd || dg) { if (d->nd < 19) { d->m = d->m * 10 + dg; --frac; } ++d->nd; }
      else --frac;
    }
  }
  if (n_int + n_frac == 0) return -1;
  long long ex = 0;
  if (s < e && (*s == 'e' || *s == 'E')) {
    ++s;
    bool eneg = false;
    if (s < e && (*s == '+' || *s == '-')) { eneg = *s == '-'; ++s; }
    if (s >= e) return -1;
    for (; s < e && is_digit(*s); ++s) ex = ex < 100000000 ? ex * 10 + (*s - '0') : ex;
    if (eneg) ex = -ex;
  }
  if (s != e) return -1;
  d->e10 = ex + frac;
  return (d->nd <= 19 && d->m <= (1ull << 53) && d->e10 >= -22 && d->e10 <= 22) ? 1 : 0;
}

__device__ __forceinline__ float fast_value(const Decimal& d) {
  double v = (double)d.m;
  v = d.e10 >= 0 ? v * kPow10[d.e10] : v / kPow10[-d.e10];
  return __double2float_rn(d.neg ? -v : v);
}

// Pass 1: count the line starts and find the first non-ASCII byte.
__global__ void obj_bytes_kernel(const uint8_t* __restrict__ b, int64_t n, unsigned long long* __restrict__ counters) {
  unsigned long long starts = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    starts += line_starts_at(b, n, i);
    if (b[i] >= 0x80) atomicMin(&counters[1], (unsigned long long)i);
  }
  for (int o = 16; o; o >>= 1) starts += __shfl_down_sync(0xffffffffu, starts, o);
  if ((threadIdx.x & 31) == 0 && starts) atomicAdd(&counters[0], starts);
}

// Pass 2 (one thread per line): the record type of the first token; vf = (is v) | (is f) << 32 for the scan, mtl = the
// line for a usemtl record else -1 (for the max-scan of parts).
__global__ void obj_classify_kernel(const uint8_t* __restrict__ b, int64_t n, const long long* __restrict__ starts,
                                    int64_t nl, uint8_t* __restrict__ type, unsigned long long* __restrict__ vf,
                                    int32_t* __restrict__ mtl) {
  const int64_t L = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (L >= nl) return;
  const uint8_t* p = b + starts[L];
  const uint8_t *tb, *te;
  uint8_t t = REC_OTHER;
  if (next_token(p, b + n, &tb, &te)) {
    const int64_t len = te - tb;
    if (len == 1 && tb[0] == 'v') t = REC_V;
    else if (len == 1 && tb[0] == 'f') t = REC_F;
    else if (len == 6 && tb[0] == 'u' && tb[1] == 's' && tb[2] == 'e' && tb[3] == 'm' && tb[4] == 't' && tb[5] == 'l')
      t = REC_MTL;
  }
  type[L] = t;
  vf[L] = (unsigned long long)(t == REC_V) | ((unsigned long long)(t == REC_F) << 32);
  if (mtl) mtl[L] = t == REC_MTL ? (int32_t)L : -1;
}

struct ParseArgs {
  const uint8_t* b;
  int64_t n;
  const long long* starts;
  int64_t nl;
  const uint8_t* type;
  const unsigned long long* vf;    // inclusive scan of (v, f) counts
  const int32_t* mtl;              // inclusive max-scan of usemtl lines, or nullptr
  int64_t nv;
  float* verts;
  int32_t* faces;
  int32_t* face_mtl;               // [nf] last usemtl line before each face (-1: none), or nullptr
  long long* slow_off;             // host-converted coordinates: token offset and vertex element
  long long* slow_dst;
  unsigned long long* counters;    // [2] status (line << 8 | reason), slow-token count
};

__device__ __forceinline__ void refuse(const ParseArgs& a, int64_t L, uint32_t why) {
  atomicMin(&a.counters[0], ((unsigned long long)L << 8) | why);
}

// Pass 3 (one thread per line): v and f records into the resident mesh.
__global__ void obj_parse_kernel(ParseArgs a) {
  const int64_t L = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (L >= a.nl) return;
  const uint8_t t = a.type[L];
  if (t != REC_V && t != REC_F) return;
  const uint8_t* p = a.b + a.starts[L];
  const uint8_t* end = a.b + a.n;
  const uint8_t *tb, *te;
  next_token(p, end, &tb, &te);                              // the record word
  if (t == REC_V) {
    const int64_t vi = (int64_t)(a.vf[L] & 0xffffffffull) - 1;
    for (int k = 0; k < 3; ++k) {
      if (!next_token(p, end, &tb, &te)) { refuse(a, L, BAD_FEW_COORDS); return; }
      Decimal d;
      const int r = scan_decimal(tb, te, &d);
      if (r < 0) { refuse(a, L, BAD_COORD); return; }
      if (r == 1) {
        a.verts[3 * vi + k] = fast_value(d);
      } else {
        const unsigned long long j = atomicAdd(&a.counters[1], 1ull);
        a.slow_off[j] = tb - a.b;
        a.slow_dst[j] = 3 * vi + k;
      }
    }
    return;
  }
  const int64_t fi = (int64_t)(a.vf[L] >> 32) - 1;
  int32_t idx[3];
  for (int k = 0; k < 3; ++k) {
    if (!next_token(p, end, &tb, &te)) { refuse(a, L, BAD_CORNERS); return; }
    const uint8_t* s = tb;
    bool neg = false;
    if (*s == '+' || *s == '-') { neg = *s == '-'; ++s; }
    long long v = 0;
    int nd = 0;
    for (; s < te && is_digit(*s); ++s, ++nd) v = v * 10 + (*s - '0');
    if (nd == 0 || nd > 18 || (s < te && *s != '/') || neg || v < 1 || v > a.nv) { refuse(a, L, BAD_INDEX); return; }
    idx[k] = (int32_t)(v - 1);
  }
  if (next_token(p, end, &tb, &te)) { refuse(a, L, BAD_CORNERS); return; }
  for (int k = 0; k < 3; ++k) a.faces[3 * fi + k] = idx[k];
  if (a.face_mtl) a.face_mtl[fi] = a.mtl[L];
}

__global__ void obj_patch_kernel(float* __restrict__ verts, const long long* __restrict__ dst,
                                 const float* __restrict__ vals, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) verts[dst[i]] = vals[i];
}

unsigned blocks_for(int64_t n) { return (unsigned)((n + OBJ_THREADS - 1) / OBJ_THREADS); }

// Device buffers of one read: the per-line arrays (c->obj_arena, sized once the line count is known) and the per-face /
// per-coordinate arrays (c->obj_lists, sized once the record counts are known).
struct ObjBufs {
  long long* starts;
  uint8_t* type;
  unsigned long long* vf;
  int32_t* mtl;
  long long* n_sel;
  void* cub_tmp;
  int32_t* face_mtl;
  long long *slow_off, *slow_dst;
  float* slow_val;
  unsigned long long* counters;   // [0] status, [1] host-converted coordinates
};

size_t carve_lines(char* base, int64_t nl, bool parts, size_t cub_bytes, ObjBufs& o) {
  Arena a{base};
  o.starts = a.take<long long>(nl);
  o.type = a.take<uint8_t>(nl);
  o.vf = a.take<unsigned long long>(nl);
  o.mtl = parts ? a.take<int32_t>(nl) : nullptr;
  o.n_sel = a.take<long long>(1);
  o.cub_tmp = a.take<char>(cub_bytes);
  return a.off;
}

size_t carve_lists(char* base, int64_t slow_cap, int64_t nf, bool parts, ObjBufs& o) {
  Arena a{base};
  o.face_mtl = parts ? a.take<int32_t>(nf) : nullptr;
  o.slow_off = a.take<long long>(slow_cap);
  o.slow_dst = a.take<long long>(slow_cap);
  o.slow_val = a.take<float>(slow_cap);
  o.counters = a.take<unsigned long long>(2);
  return a.off;
}

std::string line_message(const std::string& path, int64_t line, const std::string& why) {
  return path + ":" + std::to_string(line) + ": " + why;
}

// tokens of the line starting at byte s of the host copy
std::vector<std::string> host_tokens(const uint8_t* b, int64_t n, int64_t s) {
  std::vector<std::string> out;
  const uint8_t* p = b + s;
  const uint8_t *tb, *te;
  while (next_token(p, b + n, &tb, &te)) out.emplace_back((const char*)tb, te - tb);
  return out;
}

}  // namespace

// One coordinate token -> float32 as Python's float() then numpy's float64 -> float32 cast.  -1 outside the grammar;
// *overflow is set when a finite float64 becomes a float32 infinity.
int obj_token_to_float(const char* s, int64_t len, float* out, bool* overflow) {
  const uint8_t* b = (const uint8_t*)s;
  Decimal d;
  if (scan_decimal(b, b + len, &d) < 0) return -1;
  const char* p = s + ((*s == '+' || *s == '-') ? 1 : 0);
  const char* e = s + len;
  double v = 0.0;
  if (is_special_word((const uint8_t*)p, e - p)) {
    v = lower(*p) == 'n' ? std::nan("") : INFINITY;
  } else {
    const std::from_chars_result r = std::from_chars(p, e, v, std::chars_format::general);
    if (r.ec == std::errc::result_out_of_range) {
      // beyond double's range, where Python gives inf or 0: the value is about 10^(e10 + kept digits - 1)
      v = d.e10 + std::min(d.nd, 19) > 0 ? INFINITY : 0.0;
    } else if (r.ec != std::errc() || r.ptr != e) {
      return -1;
    }
  }
  if (d.neg) v = -v;
  const float f = (float)v;
  if (overflow && std::isfinite(v) && std::isinf(f)) *overflow = true;
  *out = f;
  return 0;
}

// Reads `path` into the resident mesh (c->mesh); see the file comment.  On success the context is in the state
// disn_mesh_load(read_obj(path)) leaves; on any failure disn_obj_read empties the resident mesh.
int obj_read(disn_ctx* c, const char* path, bool parts, int64_t* n_parts) {
  const std::string spath(path);
  auto refuse = [&](const std::string& msg) { set_error(msg); return DISN_ERR_OBJ_UNSUPPORTED; };
  c->obj_host_tokens = 0;
  c->obj_overflows = 0;
  c->obj_parts_ready = false;
  c->obj_names.clear();
  c->obj_none.clear();
  std::fill(c->obj_phase_ms, c->obj_phase_ms + 5, 0.f);

  FILE* fh = fopen(path, "rb");
  if (!fh) return refuse(spath + ": cannot open: " + strerror(errno));
  int64_t n = -1;
  if (fseeko(fh, 0, SEEK_END) == 0) n = ftello(fh);
  if (n < 0 || fseeko(fh, 0, SEEK_SET) != 0) { fclose(fh); return refuse(spath + ": cannot determine the file size"); }
  if (n >= ((int64_t)1 << 40)) { fclose(fh); return refuse(spath + ": file larger than 1 TiB"); }
  if (c->obj_host.ensure((size_t)n + 1, (size_t)n / 4) || c->obj_bytes.ensure((size_t)n + 1, (size_t)n / 4)) {
    fclose(fh);
    return -1;
  }
  uint8_t* hb = c->obj_host.as<uint8_t>();
  const size_t got = n ? fread(hb, 1, (size_t)n, fh) : 0;
  fclose(fh);
  if ((int64_t)got != n) return refuse(spath + ": short read");
  hb[n] = 0;

  for (cudaEvent_t& e : c->obj_ev)
    if (!e) DISN_CUDA_OK(cudaEventCreate(&e));
  const cudaStream_t s = c->stream;
  uint8_t* db = c->obj_bytes.as<uint8_t>();
  DISN_CUDA_OK(cudaEventRecord(c->obj_ev[0], s));
  DISN_CUDA_OK(cudaMemcpyAsync(db, hb, (size_t)n + 1, cudaMemcpyHostToDevice, s));
  DISN_CUDA_OK(cudaEventRecord(c->obj_ev[1], s));

  // line starts: count (and the first non-ASCII byte), then compact
  if (c->obj_small.ensure(4 * sizeof(unsigned long long)) || c->obj_small_host.ensure(4 * sizeof(unsigned long long)))
    return -1;
  unsigned long long* cnt = c->obj_small.as<unsigned long long>();
  unsigned long long* hcnt = c->obj_small_host.as<unsigned long long>();
  const unsigned long long init[2] = {0ull, kNoStatus};
  DISN_CUDA_OK(cudaMemcpyAsync(cnt, init, sizeof(init), cudaMemcpyHostToDevice, s));
  if (n) {
    obj_bytes_kernel<<<(unsigned)std::min<int64_t>(blocks_for(n), 8 * c->num_sms), OBJ_THREADS, 0, s>>>(db, n, cnt);
    c->launches++;
    DISN_CUDA_OK(cudaGetLastError());
  }
  DISN_CUDA_OK(cudaMemcpyAsync(hcnt, cnt, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
  DISN_CUDA_OK(cudaStreamSynchronize(s));
  const int64_t nl = (int64_t)hcnt[0];
  if (hcnt[1] != kNoStatus) {
    int64_t line = 1;
    for (int64_t i = 1; i <= (int64_t)hcnt[1]; ++i) line += line_starts_at(hb, n, i);
    return refuse(line_message(spath, line, "non-ASCII byte"));
  }
  DISN_REQUIRE(nl < ((int64_t)1 << 31), "obj_read: more than 2^31 - 1 lines");

  // scratch sized for the worst case of the vertex count (every line a v record) until the scan gives the counts
  size_t cub_bytes = 0, t = 0;
  IsLineStart pred{db, n};
  thrust::counting_iterator<long long> it(0);
  DISN_CUDA_OK(cub::DeviceSelect::If(nullptr, t, it, (long long*)nullptr, (long long*)nullptr, (long long)n, pred, s));
  cub_bytes = std::max(cub_bytes, t);
  DISN_CUDA_OK(cub::DeviceScan::InclusiveSum(nullptr, t, (unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                             (int)nl, s));
  cub_bytes = std::max(cub_bytes, t);
  DISN_CUDA_OK(cub::DeviceScan::InclusiveScan(nullptr, t, (int32_t*)nullptr, (int32_t*)nullptr, MaxOp(), (int)nl, s));
  cub_bytes = std::max(cub_bytes, t);
  ObjBufs o;
  const size_t bytes = carve_lines(nullptr, nl, parts, cub_bytes, o);
  if (c->obj_arena.ensure(bytes, bytes / 4)) return -1;
  carve_lines(c->obj_arena.as<char>(), nl, parts, cub_bytes, o);
  if (nl) {
    size_t tb = cub_bytes;
    DISN_CUDA_OK(cub::DeviceSelect::If(o.cub_tmp, tb, it, o.starts, o.n_sel, (long long)n, pred, s));
  }
  DISN_CUDA_OK(cudaEventRecord(c->obj_ev[2], s));
  if (nl) {
    obj_classify_kernel<<<blocks_for(nl), OBJ_THREADS, 0, s>>>(db, n, o.starts, nl, o.type, o.vf, o.mtl);
    c->launches++;
    DISN_CUDA_OK(cudaGetLastError());
    size_t tb = cub_bytes;
    DISN_CUDA_OK(cub::DeviceScan::InclusiveSum(o.cub_tmp, tb, o.vf, o.vf, (int)nl, s));
    if (parts) {
      tb = cub_bytes;
      DISN_CUDA_OK(cub::DeviceScan::InclusiveScan(o.cub_tmp, tb, o.mtl, o.mtl, MaxOp(), (int)nl, s));
    }
    DISN_CUDA_OK(cudaMemcpyAsync(hcnt, o.vf + nl - 1, sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
  } else {
    hcnt[0] = 0;
  }
  DISN_CUDA_OK(cudaEventRecord(c->obj_ev[3], s));
  DISN_CUDA_OK(cudaStreamSynchronize(s));
  const int64_t nv = (int64_t)(hcnt[0] & 0xffffffffull), nf = (int64_t)(hcnt[0] >> 32);
  DISN_REQUIRE(nv < ((int64_t)1 << 31) && 3 * nf < ((int64_t)1 << 31), "mesh too large for 32-bit indices");

  // parse: every v record can leave up to 3 coordinates to the host
  const int64_t slow_cap = 3 * nv;
  const size_t bytes2 = carve_lists(nullptr, slow_cap, nf, parts, o);
  if (c->obj_lists.ensure(bytes2, bytes2 / 4)) return -1;
  carve_lists(c->obj_lists.as<char>(), slow_cap, nf, parts, o);
  if (c->mesh.replace(nv, nf)) return -1;
  const unsigned long long init2[2] = {kNoStatus, 0ull};
  DISN_CUDA_OK(cudaMemcpyAsync(o.counters, init2, sizeof(init2), cudaMemcpyHostToDevice, s));
  if (nv + nf) {
    ParseArgs a{db, n, o.starts, nl, o.type, o.vf, o.mtl, nv, c->mesh.verts(), c->mesh.faces(),
                o.face_mtl, o.slow_off, o.slow_dst, o.counters};
    obj_parse_kernel<<<blocks_for(nl), OBJ_THREADS, 0, s>>>(a);
    c->launches++;
    DISN_CUDA_OK(cudaGetLastError());
  }
  DISN_CUDA_OK(cudaMemcpyAsync(hcnt, o.counters, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
  DISN_CUDA_OK(cudaEventRecord(c->obj_ev[4], s));
  DISN_CUDA_OK(cudaStreamSynchronize(s));
  if (hcnt[0] != kNoStatus) {
    const int64_t L = (int64_t)(hcnt[0] >> 8);
    const uint32_t why = (uint32_t)(hcnt[0] & 0xff);
    long long start = 0;
    DISN_CUDA_OK(cudaMemcpy(&start, o.starts + L, sizeof(start), cudaMemcpyDeviceToHost));
    std::string msg = kReason[why];
    if (why == BAD_CORNERS)
      msg += ", found " + std::to_string(host_tokens(hb, n, start).size() - 1) + " corners";
    return refuse(line_message(spath, L + 1, msg));
  }

  // host-converted coordinates
  const auto t0 = std::chrono::steady_clock::now();
  const int64_t ns = (int64_t)hcnt[1];
  c->obj_host_tokens = ns;
  if (ns) {
    if (c->obj_list_host.ensure((size_t)ns * (2 * sizeof(long long) + sizeof(float)))) return -1;
    long long* hoff = c->obj_list_host.as<long long>();
    long long* hdst = hoff + ns;
    float* hval = (float*)(hdst + ns);
    DISN_CUDA_OK(cudaMemcpyAsync(hoff, o.slow_off, ns * sizeof(long long), cudaMemcpyDeviceToHost, s));
    DISN_CUDA_OK(cudaStreamSynchronize(s));
    bool overflow = false;
    for (int64_t i = 0; i < ns; ++i) {
      const uint8_t* tb = hb + hoff[i];
      const uint8_t* te = tb;
      while (te < hb + n && !is_sep(*te) && !is_eol(*te)) ++te;
      bool of = false;
      if (obj_token_to_float((const char*)tb, te - tb, &hval[i], &of))
        return refuse(spath + ": internal error: a coordinate the device accepted was refused by the host converter");
      c->obj_overflows += of;
      overflow |= of;
    }
    DISN_CUDA_OK(cudaMemcpyAsync(o.slow_val, hval, ns * sizeof(float), cudaMemcpyHostToDevice, s));
    obj_patch_kernel<<<blocks_for(ns), OBJ_THREADS, 0, s>>>(c->mesh.verts(), o.slow_dst, o.slow_val, ns);
    c->launches++;
    DISN_CUDA_OK(cudaGetLastError());
  }

  // parts: the last usemtl line of each face -> ids numbered in order of each name's first face
  int64_t np = 0;
  if (parts) {
    if (c->obj_part_ids.ensure((size_t)std::max<int64_t>(nf, 1) * sizeof(int32_t))) return -1;
    int32_t* ids = c->obj_part_ids.as<int32_t>();
    if (nf) DISN_CUDA_OK(cudaMemcpyAsync(ids, o.face_mtl, nf * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    DISN_CUDA_OK(cudaStreamSynchronize(s));
    std::map<int32_t, int32_t> line_id;                       // usemtl line (-1: none) -> part id
    std::map<std::string, int32_t> name_id;
    int32_t none_id = -1, prev_line = INT32_MIN, prev_id = -1;
    for (int64_t f = 0; f < nf; ++f) {
      const int32_t L = ids[f];
      if (L != prev_line) {
        auto hit = line_id.find(L);
        if (hit == line_id.end()) {
          int32_t id;
          if (L < 0) {
            if (none_id < 0) { none_id = (int32_t)c->obj_names.size(); c->obj_names.push_back(""); c->obj_none.push_back(true); }
            id = none_id;
          } else {
            long long start = 0;
            DISN_CUDA_OK(cudaMemcpy(&start, o.starts + L, sizeof(start), cudaMemcpyDeviceToHost));
            const std::vector<std::string> tok = host_tokens(hb, n, start);
            const std::string name = tok.size() > 1 ? tok[1] : std::string();
            auto nh = name_id.find(name);
            if (nh == name_id.end()) {
              nh = name_id.emplace(name, (int32_t)c->obj_names.size()).first;
              c->obj_names.push_back(name);
              c->obj_none.push_back(false);
            }
            id = nh->second;
          }
          hit = line_id.emplace(L, id).first;
        }
        prev_line = L;
        prev_id = hit->second;
      }
      ids[f] = prev_id;
    }
    np = (int64_t)c->obj_names.size();
    c->obj_parts_ready = true;
    c->obj_part_faces = nf;
  }
  DISN_CUDA_OK(cudaStreamSynchronize(s));
  c->obj_phase_ms[4] = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
  for (int k = 0; k < 4; ++k) DISN_CUDA_OK(cudaEventElapsedTime(&c->obj_phase_ms[k], c->obj_ev[k], c->obj_ev[k + 1]));
  c->mesh.commit(nv, nf);
  if (n_parts) *n_parts = np;
  return 0;
}

}  // namespace disn

extern "C" {

int disn_obj_read(disn_ctx* c, const char* path, uint32_t flags, int64_t* n_verts, int64_t* n_faces, int32_t* n_parts) {
  DISN_REQUIRE(c && path, "null argument");
  DISN_REQUIRE((flags & ~(uint32_t)DISN_OBJ_PARTS) == 0, "obj_read: unknown flags");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  int64_t np = 0;
  const int rc = disn::obj_read(c, path, (flags & DISN_OBJ_PARTS) != 0, &np);
  if (rc) {
    c->obj_parts_ready = false;
    c->obj_names.clear();
    c->obj_none.clear();
  }
  if (n_parts) *n_parts = rc ? 0 : (int32_t)np;
  return disn::finish_mesh_call(c, rc, n_verts, n_faces);
}

int disn_obj_parts(disn_ctx* c, int32_t* part_ids, int64_t* name_offsets, char* names, int64_t names_capacity) {
  DISN_REQUIRE(c, "null ctx");
  DISN_REQUIRE(c->obj_parts_ready, "obj_parts: the last disn_obj_read did not succeed with DISN_OBJ_PARTS");
  const int64_t np = (int64_t)c->obj_names.size();
  int64_t total = 0;
  for (int64_t p = 0; p < np; ++p) total += (int64_t)c->obj_names[p].size();
  DISN_REQUIRE(!names || names_capacity >= total, "obj_parts: names_capacity below the names' total length");
  if (part_ids && c->obj_part_faces)
    std::memcpy(part_ids, c->obj_part_ids.as<int32_t>(), (size_t)c->obj_part_faces * sizeof(int32_t));
  int64_t off = 0;
  for (int64_t p = 0; p < np; ++p) {
    const std::string& nm = c->obj_names[p];
    if (name_offsets) name_offsets[p] = c->obj_none[p] ? -1 : off;
    if (names && !nm.empty()) std::memcpy(names + off, nm.data(), nm.size());
    off += (int64_t)nm.size();
  }
  if (name_offsets) name_offsets[np] = off;
  return 0;
}

int disn_obj_read_stats(disn_ctx* c, int64_t* counts, float* phase_ms) {
  DISN_REQUIRE(c, "null ctx");
  if (counts) { counts[0] = c->obj_host_tokens; counts[1] = c->obj_overflows; }
  if (phase_ms) std::memcpy(phase_ms, c->obj_phase_ms, sizeof(c->obj_phase_ms));
  return 0;
}

}  // extern "C"
