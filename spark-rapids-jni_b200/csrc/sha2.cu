// sha2.cu -- Hash.sha{224,256,384,512}NullsPreserved (reference hash/sha.cpp:31-49 over cudf's sha_hash.cuh): FIPS 180-4
// SHA-2 of every row of a STRING column, written as lowercase hex into a STRING column that keeps the input's nulls.
//
// One lane hashes one row (a warp = 32 consecutive rows).  The message words come from 4-byte aligned loads of the chars,
// funnel-shifted to the string's byte alignment and byte-swapped to big-endian; the 0x80 / length padding is built in
// registers.  The rounds are fully unrolled over a rolling 16-word schedule window; round constants live in __constant__
// (one c[][] operand per round).  SHA-224 / SHA-384 are the SHA-256 / SHA-512 kernels with other initial values and a
// truncated digest.  A null row (mask bit clear) gets no chars: its output offsets are equal (purge_nonempty_nulls).
#include "check.hpp"
#include "common.cuh"
#include "kernels.hpp"

namespace srj {
namespace {

constexpr int kShaThreads = 256;

__constant__ uint32_t kK256[64] = {
  0x428a2f98u, 0x71374491u, 0xb5c0fbcfu, 0xe9b5dba5u, 0x3956c25bu, 0x59f111f1u, 0x923f82a4u, 0xab1c5ed5u,
  0xd807aa98u, 0x12835b01u, 0x243185beu, 0x550c7dc3u, 0x72be5d74u, 0x80deb1feu, 0x9bdc06a7u, 0xc19bf174u,
  0xe49b69c1u, 0xefbe4786u, 0x0fc19dc6u, 0x240ca1ccu, 0x2de92c6fu, 0x4a7484aau, 0x5cb0a9dcu, 0x76f988dau,
  0x983e5152u, 0xa831c66du, 0xb00327c8u, 0xbf597fc7u, 0xc6e00bf3u, 0xd5a79147u, 0x06ca6351u, 0x14292967u,
  0x27b70a85u, 0x2e1b2138u, 0x4d2c6dfcu, 0x53380d13u, 0x650a7354u, 0x766a0abbu, 0x81c2c92eu, 0x92722c85u,
  0xa2bfe8a1u, 0xa81a664bu, 0xc24b8b70u, 0xc76c51a3u, 0xd192e819u, 0xd6990624u, 0xf40e3585u, 0x106aa070u,
  0x19a4c116u, 0x1e376c08u, 0x2748774cu, 0x34b0bcb5u, 0x391c0cb3u, 0x4ed8aa4au, 0x5b9cca4fu, 0x682e6ff3u,
  0x748f82eeu, 0x78a5636fu, 0x84c87814u, 0x8cc70208u, 0x90befffau, 0xa4506cebu, 0xbef9a3f7u, 0xc67178f2u};

__constant__ uint64_t kK512[80] = {
  0x428a2f98d728ae22ull, 0x7137449123ef65cdull, 0xb5c0fbcfec4d3b2full, 0xe9b5dba58189dbbcull, 0x3956c25bf348b538ull,
  0x59f111f1b605d019ull, 0x923f82a4af194f9bull, 0xab1c5ed5da6d8118ull, 0xd807aa98a3030242ull, 0x12835b0145706fbeull,
  0x243185be4ee4b28cull, 0x550c7dc3d5ffb4e2ull, 0x72be5d74f27b896full, 0x80deb1fe3b1696b1ull, 0x9bdc06a725c71235ull,
  0xc19bf174cf692694ull, 0xe49b69c19ef14ad2ull, 0xefbe4786384f25e3ull, 0x0fc19dc68b8cd5b5ull, 0x240ca1cc77ac9c65ull,
  0x2de92c6f592b0275ull, 0x4a7484aa6ea6e483ull, 0x5cb0a9dcbd41fbd4ull, 0x76f988da831153b5ull, 0x983e5152ee66dfabull,
  0xa831c66d2db43210ull, 0xb00327c898fb213full, 0xbf597fc7beef0ee4ull, 0xc6e00bf33da88fc2ull, 0xd5a79147930aa725ull,
  0x06ca6351e003826full, 0x142929670a0e6e70ull, 0x27b70a8546d22ffcull, 0x2e1b21385c26c926ull, 0x4d2c6dfc5ac42aedull,
  0x53380d139d95b3dfull, 0x650a73548baf63deull, 0x766a0abb3c77b2a8ull, 0x81c2c92e47edaee6ull, 0x92722c851482353bull,
  0xa2bfe8a14cf10364ull, 0xa81a664bbc423001ull, 0xc24b8b70d0f89791ull, 0xc76c51a30654be30ull, 0xd192e819d6ef5218ull,
  0xd69906245565a910ull, 0xf40e35855771202aull, 0x106aa07032bbd1b8ull, 0x19a4c116b8d2d0c8ull, 0x1e376c085141ab53ull,
  0x2748774cdf8eeb99ull, 0x34b0bcb5e19b48a8ull, 0x391c0cb3c5c95a63ull, 0x4ed8aa4ae3418acbull, 0x5b9cca4f7763e373ull,
  0x682e6ff3d6b2b8a3ull, 0x748f82ee5defb2fcull, 0x78a5636f43172f60ull, 0x84c87814a1f0ab72ull, 0x8cc702081a6439ecull,
  0x90befffa23631e28ull, 0xa4506cebde82bde9ull, 0xbef9a3f7b2c67915ull, 0xc67178f2e372532bull, 0xca273eceea26619cull,
  0xd186b8c721c0c207ull, 0xeada7dd6cde0eb1eull, 0xf57d4f7fee6ed178ull, 0x06f067aa72176fbaull, 0x0a637dc5a2c898a6ull,
  0x113f9804bef90daeull, 0x1b710b35131c471bull, 0x28db77f523047d84ull, 0x32caab7b40c72493ull, 0x3c9ebe0a15c9bebcull,
  0x431d67c49c100d4cull, 0x4cc5d4becb3e42b6ull, 0x597f299cfc657e2aull, 0x5fcb6fab3ad6faecull, 0x6c44198c4a475817ull};

// initial hash values (FIPS 180-4 §5.3)
__constant__ uint32_t kIV224[8] = {0xc1059ed8u, 0x367cd507u, 0x3070dd17u, 0xf70e5939u, 0xffc00b31u, 0x68581511u, 0x64f98fa7u, 0xbefa4fa4u};
__constant__ uint32_t kIV256[8] = {0x6a09e667u, 0xbb67ae85u, 0x3c6ef372u, 0xa54ff53au, 0x510e527fu, 0x9b05688cu, 0x1f83d9abu, 0x5be0cd19u};
__constant__ uint64_t kIV384[8] = {0xcbbb9d5dc1059ed8ull, 0x629a292a367cd507ull, 0x9159015a3070dd17ull, 0x152fecd8f70e5939ull,
                                   0x67332667ffc00b31ull, 0x8eb44a8768581511ull, 0xdb0c2e0d64f98fa7ull, 0x47b5481dbefa4fa4ull};
__constant__ uint64_t kIV512[8] = {0x6a09e667f3bcc908ull, 0xbb67ae8584caa73bull, 0x3c6ef372fe94f82bull, 0xa54ff53a5f1d36f1ull,
                                   0x510e527fade682d1ull, 0x9b05688c2b3e6c1full, 0x1f83d9abfb41bd6bull, 0x5be0cd19137e2179ull};

__device__ __forceinline__ uint32_t rotr32(uint32_t x, int n) { return __funnelshift_r(x, x, n); }

// 64-bit rotate as two funnel shifts on the halves (n is a compile-time constant in every use)
__device__ __forceinline__ uint64_t rotr64(uint64_t x, int n)
{
  const uint32_t lo = static_cast<uint32_t>(x), hi = static_cast<uint32_t>(x >> 32);
  uint32_t rlo, rhi;
  if (n < 32) { rlo = __funnelshift_r(lo, hi, n); rhi = __funnelshift_r(hi, lo, n); }
  else        { rlo = __funnelshift_r(hi, lo, n - 32); rhi = __funnelshift_r(lo, hi, n - 32); }
  return (static_cast<uint64_t>(rhi) << 32) | rlo;
}

// Big-endian 32-bit message words [bpos, bpos + 4 * NW) of a string of `len` bytes, with the 0x80 terminator and zero
// padding past its end.  `aw` = the 4-byte aligned word holding the string's first byte, `r` = that byte's position in it.
// Only aligned words holding at least one byte of the string are loaded.
template <int NW>
__device__ __forceinline__ void message_words(const uint32_t* aw, int r, int32_t len, int32_t bpos, uint32_t (&m)[NW])
{
  uint32_t A[NW + 1];
  const uint32_t* p = aw + bpos / 4;
#pragma unroll
  for (int k = 0; k <= NW; ++k) A[k] = bpos + 4 * k - r < len ? __ldg(p + k) : 0u;
#pragma unroll
  for (int i = 0; i < NW; ++i) {
    const uint32_t w = __byte_perm(__funnelshift_r(A[i], A[i + 1], 8 * r), 0u, 0x0123);
    const int32_t d  = len - (bpos + 4 * i);   // string bytes left at this word
    m[i] = d >= 4 ? w : d >= 0 ? (w & ~(0xffffffffu >> (8 * d))) | (0x80000000u >> (8 * d)) : 0u;
  }
}

__device__ __forceinline__ void sha256_compress(uint32_t (&st)[8], uint32_t (&w)[16])
{
  uint32_t a = st[0], b = st[1], c = st[2], d = st[3], e = st[4], f = st[5], g = st[6], h = st[7];
#pragma unroll
  for (int t = 0; t < 64; ++t) {
    if (t >= 16) {
      const uint32_t x = w[(t - 15) & 15], y = w[(t - 2) & 15];
      w[t & 15] += (rotr32(x, 7) ^ rotr32(x, 18) ^ (x >> 3)) + w[(t - 7) & 15] + (rotr32(y, 17) ^ rotr32(y, 19) ^ (y >> 10));
    }
    const uint32_t t1 = h + (rotr32(e, 6) ^ rotr32(e, 11) ^ rotr32(e, 25)) + ((e & f) ^ (~e & g)) + kK256[t] + w[t & 15];
    const uint32_t t2 = (rotr32(a, 2) ^ rotr32(a, 13) ^ rotr32(a, 22)) + ((a & b) ^ (a & c) ^ (b & c));
    h = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
  }
  st[0] += a; st[1] += b; st[2] += c; st[3] += d; st[4] += e; st[5] += f; st[6] += g; st[7] += h;
}

__device__ __forceinline__ void sha512_compress(uint64_t (&st)[8], uint64_t (&w)[16])
{
  uint64_t a = st[0], b = st[1], c = st[2], d = st[3], e = st[4], f = st[5], g = st[6], h = st[7];
#pragma unroll
  for (int t = 0; t < 80; ++t) {
    if (t >= 16) {
      const uint64_t x = w[(t - 15) & 15], y = w[(t - 2) & 15];
      w[t & 15] += (rotr64(x, 1) ^ rotr64(x, 8) ^ (x >> 7)) + w[(t - 7) & 15] + (rotr64(y, 19) ^ rotr64(y, 61) ^ (y >> 6));
    }
    const uint64_t t1 = h + (rotr64(e, 14) ^ rotr64(e, 18) ^ rotr64(e, 41)) + ((e & f) ^ (~e & g)) + kK512[t] + w[t & 15];
    const uint64_t t2 = (rotr64(a, 28) ^ rotr64(a, 34) ^ rotr64(a, 39)) + ((a & b) ^ (a & c) ^ (b & c));
    h = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
  }
  st[0] += a; st[1] += b; st[2] += c; st[3] += d; st[4] += e; st[5] += f; st[6] += g; st[7] += h;
}

// 8 lowercase hex chars of a big-endian word, as two little-endian words of chars: nibble -> ASCII four bytes at a time
// ('0' + n, plus 39 when n > 9: bit 4 of n + 6 says so), then one byte permute per output word interleaves hi / lo.
__device__ __forceinline__ uint2 hex8(uint32_t x)
{
  const uint32_t hi = (x >> 4) & 0x0f0f0f0fu, lo = x & 0x0f0f0f0fu;
  const uint32_t H  = hi + 0x30303030u + (((hi + 0x06060606u) >> 4) & 0x01010101u) * 0x27u;
  const uint32_t L  = lo + 0x30303030u + (((lo + 0x06060606u) >> 4) & 0x01010101u) * 0x27u;
  return make_uint2(__byte_perm(H, L, 0x6273), __byte_perm(H, L, 0x4051));
}

// D digest words -> 8 * D chars at dst: 16-byte stores when the row's width (and so its offset rank * width) is a multiple
// of 16, else 8-byte stores (SHA-224: 56 chars)
template <int D>
__device__ __forceinline__ void store_hex(uint8_t* dst, const uint32_t (&dig)[D])
{
  if constexpr (D % 2 == 0) {
#pragma unroll
    for (int i = 0; i < D / 2; ++i) {
      const uint2 a = hex8(dig[2 * i]), b = hex8(dig[2 * i + 1]);
      *reinterpret_cast<uint4*>(dst + 16 * i) = make_uint4(a.x, a.y, b.x, b.y);
    }
  } else {
#pragma unroll
    for (int i = 0; i < D; ++i) *reinterpret_cast<uint2*>(dst + 8 * i) = hex8(dig[i]);
  }
}

struct RowRef {
  const uint32_t* aw;
  int r;
  int32_t len;
  uint8_t* dst;
};

// the row this lane hashes, or false for a null row / a lane past the end
__device__ __forceinline__ bool row_ref(const uint8_t* chars, const int32_t* in_off, const uint32_t* mask, int64_t n, const int32_t* out_off,
                                        uint8_t* out_chars, RowRef* rr)
{
  const int64_t row = static_cast<int64_t>(blockIdx.x) * kShaThreads + threadIdx.x;
  if (row >= n) return false;
  if (mask && !((__ldg(mask + (row >> 5)) >> (row & 31)) & 1u)) return false;
  const int32_t beg = __ldg(in_off + row);
  const uint8_t* s  = chars + beg;
  rr->aw  = reinterpret_cast<const uint32_t*>(reinterpret_cast<uintptr_t>(s) & ~uintptr_t{3});
  rr->r   = static_cast<int>(reinterpret_cast<uintptr_t>(s) & 3);
  rr->len = __ldg(in_off + row + 1) - beg;
  rr->dst = out_chars + __ldg(out_off + row);
  return true;
}

template <bool k224>
__global__ void __launch_bounds__(kShaThreads) sha256_kernel(const uint8_t* __restrict__ chars, const int32_t* __restrict__ in_off,
                                                           const uint32_t* __restrict__ mask, int64_t n, const int32_t* __restrict__ out_off,
                                                           uint8_t* __restrict__ out_chars)
{
  RowRef rr;
  if (!row_ref(chars, in_off, mask, n, out_off, out_chars, &rr)) return;
  uint32_t st[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) st[i] = k224 ? kIV224[i] : kIV256[i];
  const int32_t nblk = (rr.len + 8) / 64 + 1;   // message + 0x80 + 8-byte length
  for (int32_t b = 0; b < nblk; ++b) {
    uint32_t w[16];
    message_words<16>(rr.aw, rr.r, rr.len, 64 * b, w);
    if (b == nblk - 1) {
      w[14] = static_cast<uint32_t>(rr.len) >> 29;
      w[15] = static_cast<uint32_t>(rr.len) << 3;
    }
    sha256_compress(st, w);
  }
  constexpr int D = k224 ? 7 : 8;
  uint32_t dig[D];
#pragma unroll
  for (int i = 0; i < D; ++i) dig[i] = st[i];
  store_hex<D>(rr.dst, dig);
}

template <bool k384>
__global__ void __launch_bounds__(kShaThreads) sha512_kernel(const uint8_t* __restrict__ chars, const int32_t* __restrict__ in_off,
                                                           const uint32_t* __restrict__ mask, int64_t n, const int32_t* __restrict__ out_off,
                                                           uint8_t* __restrict__ out_chars)
{
  RowRef rr;
  if (!row_ref(chars, in_off, mask, n, out_off, out_chars, &rr)) return;
  uint64_t st[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) st[i] = k384 ? kIV384[i] : kIV512[i];
  const int32_t nblk = (rr.len + 16) / 128 + 1;  // message + 0x80 + 16-byte length
  for (int32_t b = 0; b < nblk; ++b) {
    uint32_t m[32];
    message_words<32>(rr.aw, rr.r, rr.len, 128 * b, m);
    if (b == nblk - 1) {                         // the length's upper 64 bits are zero (len < 2^31)
      m[30] = static_cast<uint32_t>(rr.len) >> 29;
      m[31] = static_cast<uint32_t>(rr.len) << 3;
    }
    uint64_t w[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) w[i] = (static_cast<uint64_t>(m[2 * i]) << 32) | m[2 * i + 1];
    sha512_compress(st, w);
  }
  constexpr int D = k384 ? 12 : 16;
  uint32_t dig[D];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) {
    dig[2 * i]     = static_cast<uint32_t>(st[i] >> 32);
    dig[2 * i + 1] = static_cast<uint32_t>(st[i]);
  }
  store_hex<D>(rr.dst, dig);
}

// ---- output offsets ------------------------------------------------------------------------------------------------
// rank[w] = valid rows of mask word w (bits past row n - 1 ignored)
__global__ void __launch_bounds__(kShaThreads) sha2_word_popc_kernel(const uint32_t* __restrict__ mask, int64_t n, int32_t* __restrict__ rank)
{
  const int64_t w = static_cast<int64_t>(blockIdx.x) * kShaThreads + threadIdx.x;
  if (w >= (n + 31) / 32) return;
  uint32_t m        = mask[w];
  const int64_t rem = n - 32 * w;
  if (rem < 32) m &= (1u << rem) - 1u;
  rank[w] = __popc(m);
}

// offsets[r] = width x (valid rows before r); rank = exclusive scan of the word counts, rank[words] = valid rows in all.
// Without a mask every row is valid: offsets[r] = width x r.
__global__ void __launch_bounds__(kShaThreads) sha2_offsets_kernel(const uint32_t* __restrict__ mask, const int32_t* __restrict__ rank, int64_t n,
                                                                 int32_t width, int32_t* __restrict__ offsets)
{
  const int64_t r = static_cast<int64_t>(blockIdx.x) * kShaThreads + threadIdx.x;
  if (r > n) return;
  int64_t valid_before;
  if (!mask) valid_before = r;
  else if (r == n) valid_before = rank[(n + 31) / 32];
  else valid_before = rank[r >> 5] + __popc(mask[r >> 5] & ((1u << (r & 31)) - 1u));
  offsets[r] = static_cast<int32_t>(width * valid_before);
}

}  // namespace

static int32_t sha2_hex_width(int32_t digest_bits)
{
  switch (digest_bits) {
    case 224: return 56;
    case 256: return 64;
    case 384: return 96;
    case 512: return 128;
    default: return 0;
  }
}

// [rank: words + 1 ints | scan sums]
static int64_t sha2_workspace_bytes(int64_t n)
{
  const int64_t words = (n + 31) / 32;
  return 4 * (words + 1 + i32_scan_nchunks(words));
}

static int launch_sha2_sizes(int32_t digest_bits, const srj_column& in, int32_t* d_offsets, int64_t* h_total, void* workspace, cudaStream_t stream)
{
  const int64_t n     = in.size;
  const int32_t width = sha2_hex_width(digest_bits);
  const unsigned grid = static_cast<unsigned>((n + 1 + kShaThreads - 1) / kShaThreads);
  if (!in.null_mask || n == 0) {
    *h_total = width * n;
    if (*h_total > INT32_MAX) return SRJ_EOVERFLOW;   // checked before anything is written: no sync needed
    sha2_offsets_kernel<<<grid, kShaThreads, 0, stream>>>(nullptr, nullptr, n, width, d_offsets);
    SRJ_CUDA_TRY(cudaGetLastError());
    return SRJ_OK;
  }
  const int64_t words = (n + 31) / 32;
  auto* rank          = static_cast<int32_t*>(workspace);
  sha2_word_popc_kernel<<<static_cast<unsigned>((words + kShaThreads - 1) / kShaThreads), kShaThreads, 0, stream>>>(in.null_mask, n, rank);
  SRJ_CUDA_TRY(cudaGetLastError());
  int rc = launch_i32_exclusive_scan(rank, words, rank + words + 1, rank + words, stream);
  if (rc != SRJ_OK) return rc;
  int32_t valid = 0;
  SRJ_CUDA_TRY(cudaMemcpyAsync(&valid, rank + words, 4, cudaMemcpyDeviceToHost, stream));
  SRJ_CUDA_TRY(cudaStreamSynchronize(stream));
  *h_total = static_cast<int64_t>(width) * valid;
  if (*h_total > INT32_MAX) return SRJ_EOVERFLOW;
  sha2_offsets_kernel<<<grid, kShaThreads, 0, stream>>>(in.null_mask, rank, n, width, d_offsets);
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

static int launch_sha2(int32_t digest_bits, const srj_column& in, const srj_column& out, cudaStream_t stream)
{
  const int64_t n = in.size;
  if (n == 0) return SRJ_OK;
  const size_t mask_bytes = static_cast<size_t>((n + 31) / 32) * 4;
  if (out.null_mask) {
    if (in.null_mask) SRJ_CUDA_TRY(cudaMemcpyAsync(out.null_mask, in.null_mask, mask_bytes, cudaMemcpyDeviceToDevice, stream));
    else SRJ_CUDA_TRY(cudaMemsetAsync(out.null_mask, 0xff, mask_bytes, stream));
  }
  const unsigned grid = static_cast<unsigned>((n + kShaThreads - 1) / kShaThreads);
  auto* chars         = static_cast<const uint8_t*>(in.data);
  auto* out_chars     = static_cast<uint8_t*>(out.data);
  switch (digest_bits) {
    case 224: sha256_kernel<true><<<grid, kShaThreads, 0, stream>>>(chars, in.offsets, in.null_mask, n, out.offsets, out_chars); break;
    case 256: sha256_kernel<false><<<grid, kShaThreads, 0, stream>>>(chars, in.offsets, in.null_mask, n, out.offsets, out_chars); break;
    case 384: sha512_kernel<true><<<grid, kShaThreads, 0, stream>>>(chars, in.offsets, in.null_mask, n, out.offsets, out_chars); break;
    default: sha512_kernel<false><<<grid, kShaThreads, 0, stream>>>(chars, in.offsets, in.null_mask, n, out.offsets, out_chars); break;
  }
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

}  // namespace srj

// ---- C ABI (include/srj_b200.h) ----
using namespace srj;

extern "C" {

int64_t srj_sha2_workspace_bytes(int64_t num_rows) { return sha2_workspace_bytes(std::max<int64_t>(0, num_rows)); }

static int sha2_check(const char* what, int32_t digest_bits, const srj_column* in)
{
  if (sha2_hex_width(digest_bits) == 0) { set_error("%s: digest_bits %d is not one of 224, 256, 384, 512", what, digest_bits); return SRJ_EINVAL; }
  if (!in) { set_error("%s: input is null", what); return SRJ_EINVAL; }
  if (in->type_id != SRJ_STRING) { set_error("%s: SHA-2 hashing requires a string column (type id %d)", what, in->type_id); return SRJ_EUNSUPPORTED; }
  if (in->size < 0 || in->size > INT32_MAX) { set_error("%s: %lld rows", what, static_cast<long long>(in->size)); return SRJ_EINVAL; }
  if (in->size > 0 && !in->offsets) { set_error("%s: the STRING column has no offsets", what); return SRJ_EINVAL; }
  return SRJ_OK;
}

int srj_sha2_sizes(int32_t digest_bits, const srj_column* input, int32_t* d_out_offsets, int64_t* total_chars, void* workspace, void* stream)
{
  SRJ_API_RANGE();
  int rc = sha2_check("sha2_sizes", digest_bits, input);
  if (rc != SRJ_OK) return rc;
  if (!d_out_offsets || !total_chars) { set_error("sha2_sizes: bad argument"); return SRJ_EINVAL; }
  if (input->null_mask && input->size > 0 && !workspace) { set_error("sha2_sizes: an input with a null mask needs the workspace (srj_sha2_workspace_bytes)"); return SRJ_EINVAL; }
  rc = launch_sha2_sizes(digest_bits, *input, d_out_offsets, total_chars, workspace, static_cast<cudaStream_t>(stream));
  if (rc == SRJ_EOVERFLOW)
    set_error("sha2_sizes: %lld chars of SHA-%d hex exceed one STRING column (INT32_MAX): hash fewer rows per call", static_cast<long long>(*total_chars), digest_bits);
  return rc;
}

int srj_sha2_hash(int32_t digest_bits, const srj_column* input, const srj_column* out, void* stream)
{
  SRJ_API_RANGE();
  int rc = sha2_check("sha2_hash", digest_bits, input);
  if (rc != SRJ_OK) return rc;
  if (!out || out->size != input->size || (input->size > 0 && !out->offsets)) { set_error("sha2_hash: the output needs the offsets of srj_sha2_sizes and the input's row count"); return SRJ_EINVAL; }
  const bool nulls = input->null_mask && input->size > 0;
  if ((rc = check_out("sha2_hash", "output mask", out->null_mask, 1, nulls)) != SRJ_OK) return rc;
  if ((rc = check_out("sha2_hash", "output chars", out->data, 16, !input->null_mask && input->size > 0)) != SRJ_OK) return rc;
  return launch_sha2(digest_bits, *input, *out, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
