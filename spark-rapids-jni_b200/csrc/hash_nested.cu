// hash_nested.cu -- Spark row hashes over tables with LIST / STRUCT key columns (reference: the nested branches of
// hash/xxhash64.cu:446-506, hash/murmur_hash.cu:119-144, hash/hive_hash.cu:363-433; depth limits
// xxhash64.cu:513-543, hive_hash.cu:441-466, MAX_STACK_DEPTH = 8 hash/hash.hpp:28).
//
// The column trees are flattened on the host into one node table (a small per-call upload); a thread hashes a row by
// walking the tree of each key column with an explicit stack -- no recursion, no per-row allocation:
//   xxhash64 / murmur3 : the leaf values under the row are chained depth first (a LIST contributes the elements its
//                        offsets select, a STRUCT its fields in order, element by element); a null leaf keeps the
//                        accumulator; xxhash64 does not look at list / struct level nulls (xxhash64.cu:460-462),
//                        murmur3 skips a null list or struct element with everything under it (see chain_nested);
//   hive               : h(struct) = fold 31 * h + h(field), h(list) = fold 31 * h + h(element), null leaf -> 0.
// Nested keys are the uncommon case of shuffle partitioning: this kernel is one row per thread and serves correctness;
// flat keys never come here (hash.cu).
#include <algorithm>
#include <cstring>
#include <type_traits>
#include <vector>

#include "check.hpp"
#include "common.cuh"
#include "hash_device.cuh"
#include "kernels.hpp"

namespace srj {

struct HNode {
  const uint8_t* data;
  const uint32_t* mask;
  const int32_t* offsets;
  int32_t type;
  int32_t size;         // bytes per element (0: STRING / LIST / STRUCT)
  int32_t first_child;  // index of the first child node (children are consecutive)
  int32_t num_children;
};

constexpr int kNestStack   = SRJ_MAX_STACK_DEPTH + 2;
constexpr int kMurmurStack = 2 * SRJ_MAX_STACK_DEPTH + 2;   // murmur3 also keeps a frame per nullable LIST level

__device__ __forceinline__ bool node_valid(const HNode& n, int64_t i) { return !n.mask || ((n.mask[i >> 5] >> (i & 31)) & 1u); }

__device__ __forceinline__ void leaf_value(const HNode& n, int64_t i, uint64_t& v, uint64_t& v2)
{
  v2 = 0;
  const uint8_t* p = n.data + i * n.size;
  switch (n.size) {
    case 1: v = *p; break;
    case 2: v = *reinterpret_cast<const uint16_t*>(p); break;
    case 4: v = *reinterpret_cast<const uint32_t*>(p); break;
    case 8: v = *reinterpret_cast<const unsigned long long*>(p); break;
    default:
      v  = reinterpret_cast<const unsigned long long*>(p)[0];
      v2 = reinterpret_cast<const unsigned long long*>(p)[1];
  }
}

template <int KIND, class acc_t>
__device__ __forceinline__ acc_t chain_leaf(const HNode& n, int64_t i, acc_t h)
{
  if (!node_valid(n, i)) return h;
  if (n.type == SRJ_STRING) {
    const int32_t o0 = n.offsets[i], o1 = n.offsets[i + 1];
    if constexpr (KIND == SRJ_HASH_XXHASH64) return hash::xx_bytes(n.data + o0, o1 - o0, h);
    else return hash::mm_bytes(n.data + o0, o1 - o0, h);
  }
  uint64_t v, v2;
  leaf_value(n, i, v, v2);
  if constexpr (KIND == SRJ_HASH_XXHASH64) return hash::xx_fixed(n.type, v, v2, h);
  else return hash::mm_fixed(n.type, v, v2, h);
}

__device__ __forceinline__ uint32_t hive_leaf(const HNode& n, int64_t i)
{
  if (!node_valid(n, i)) return 0u;
  if (n.type == SRJ_STRING) {
    const int32_t o0 = n.offsets[i], o1 = n.offsets[i + 1];
    return static_cast<uint32_t>(hash::hive_bytes(n.data + o0, o1 - o0));
  }
  uint64_t v, v2;
  leaf_value(n, i, v, v2);
  return static_cast<uint32_t>(hash::hive_fixed(n.type, v));
}

__device__ __forceinline__ bool is_nested(int32_t t) { return t == SRJ_LIST || t == SRJ_STRUCT; }

// xxhash64 / murmur3: chain every leaf under element range [lo, hi) of `root`.
// xxhash64 does not look at LIST / STRUCT level nulls (xxhash64.cu:460-462).  murmur3 runs on the table cudf's row
// hasher prepared (murmur_hash.cu:210): struct nulls pushed down into the fields, null list rows emptied
// (cudf row_operators.cu:845-852), so a null LIST or STRUCT element contributes nothing.
template <int KIND, class acc_t>
__device__ acc_t chain_nested(const HNode* nodes, int root, int64_t row, acc_t h)
{
  constexpr bool kLevelNulls = KIND == SRJ_HASH_MURMUR3_32;
  constexpr int kStack       = kLevelNulls ? kMurmurStack : kNestStack;
  struct Frame { int32_t node, child; int64_t i, hi; };
  Frame st[kStack];
  int sp = 0;
  st[sp++] = Frame{root, 0, row, row + 1};
  while (sp > 0) {
    Frame& f       = st[sp - 1];
    const HNode& n = nodes[f.node];
    if (n.type == SRJ_LIST) {
      if (!kLevelNulls || !n.mask) {
        // a list is replaced by the elements its offsets select (nested lists collapse level by level)
        const int64_t lo = n.offsets[f.i], hi = n.offsets[f.hi];
        f = Frame{n.first_child, 0, lo, hi};
      } else {
        // a nullable list under murmur3: its rows one at a time, the elements of each valid row in a frame above
        if (f.i >= f.hi) { --sp; continue; }
        const int64_t i = f.i++;
        if (node_valid(n, i) && sp < kStack) st[sp++] = Frame{n.first_child, 0, n.offsets[i], n.offsets[i + 1]};
      }
    } else if (n.type == SRJ_STRUCT) {
      if (f.i >= f.hi) { --sp; continue; }
      if (f.child == n.num_children) { ++f.i; f.child = 0; continue; }
      if (kLevelNulls && f.child == 0 && !node_valid(n, f.i)) { ++f.i; continue; }
      const int c = n.first_child + f.child++;
      if (sp < kStack) st[sp++] = Frame{c, 0, f.i, f.i + 1};   // depth was checked on the host
    } else {
      for (int64_t i = f.i; i < f.hi; ++i) h = chain_leaf<KIND>(n, i, h);
      --sp;
    }
  }
  return h;
}

// hive: structural hash of element `row` of `root`
__device__ uint32_t hive_nested(const HNode* nodes, int root, int64_t row)
{
  struct Frame { int32_t node; int32_t pad; int64_t idx, cur, end; uint32_t acc; };
  Frame st[kNestStack];
  int sp         = 0;
  uint32_t result = 0;
  auto push = [&](int node, int64_t idx) {
    const HNode& n = nodes[node];
    Frame f{node, 0, idx, 0, 0, 0u};
    if (n.type == SRJ_LIST) { f.cur = n.offsets[idx]; f.end = n.offsets[idx + 1]; }
    else { f.cur = 0; f.end = n.num_children; }
    st[sp++] = f;
  };
  auto deliver = [&](uint32_t v) {
    --sp;
    if (sp == 0) result = v;
    else st[sp - 1].acc = 31u * st[sp - 1].acc + v;
  };
  push(root, row);
  while (sp > 0) {
    Frame& f       = st[sp - 1];
    const HNode& n = nodes[f.node];
    if (f.cur >= f.end) { deliver(f.acc); continue; }
    if (n.type == SRJ_STRUCT) {
      const int c     = n.first_child + static_cast<int>(f.cur++);
      const HNode& cn = nodes[c];
      if (!is_nested(cn.type)) f.acc = 31u * f.acc + hive_leaf(cn, f.idx);
      else if (sp < kNestStack) push(c, f.idx);
    } else {  // LIST
      const HNode& cn = nodes[n.first_child];
      if (!is_nested(cn.type)) {
        for (; f.cur < f.end; ++f.cur) f.acc = 31u * f.acc + hive_leaf(cn, f.cur);
      } else if (sp < kNestStack) {
        push(n.first_child, f.cur++);
      }
    }
  }
  return result;
}

template <int KIND>
__global__ void __launch_bounds__(256) row_hash_nested_kernel(const HNode* nodes, const int32_t* roots, int nroots, int64_t n,
                                                               int64_t seed, void* out)
{
  const int64_t r = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (r >= n) return;
  if constexpr (KIND == SRJ_HASH_HIVE) {
    uint32_t h = 0;
    for (int c = 0; c < nroots; ++c) {
      const HNode& nd = nodes[roots[c]];
      const uint32_t x = is_nested(nd.type) ? hive_nested(nodes, roots[c], r) : hive_leaf(nd, r);
      h = 31u * h + x;   // hive_hash.cu:179-191
    }
    reinterpret_cast<uint32_t*>(out)[r] = h;
  } else {
    using acc_t = typename std::conditional<KIND == SRJ_HASH_XXHASH64, uint64_t, uint32_t>::type;
    acc_t h     = static_cast<acc_t>(seed);
    for (int c = 0; c < nroots; ++c) {
      const HNode& nd = nodes[roots[c]];
      h = is_nested(nd.type) ? chain_nested<KIND>(nodes, roots[c], r, h) : chain_leaf<KIND>(nd, r, h);
    }
    reinterpret_cast<acc_t*>(out)[r] = h;
  }
}

// ---- host side ---------------------------------------------------------------------------------------------------
// depth rules of the reference: xxhash64.cu:513-543 (a LIST of STRUCT counts one extra level; leaves count 1),
// hive_hash.cu:441-466 (every LIST / STRUCT level counts 1, leaves 0); murmur has no limit of its own (recursion-free
// because structs are decomposed up front) -- the xxhash64 rule is applied to it as well.
static int depth_xx(const srj_column& c)
{
  if (c.type_id == SRJ_LIST) {
    if (c.num_children < 1) return 1;
    const srj_column& ch = c.children[0];
    return (ch.type_id == SRJ_STRUCT ? 1 : 0) + depth_xx(ch);
  }
  if (c.type_id == SRJ_STRUCT) {
    int m = 0;
    for (int i = 0; i < c.num_children; ++i) m = std::max(m, depth_xx(c.children[i]));
    return 1 + m;
  }
  return 1;
}
static int depth_hive(const srj_column& c)
{
  if (c.type_id == SRJ_LIST) return 1 + (c.num_children > 0 ? depth_hive(c.children[0]) : 0);
  if (c.type_id == SRJ_STRUCT) {
    int m = 0;
    for (int i = 0; i < c.num_children; ++i) m = std::max(m, depth_hive(c.children[i]));
    return 1 + m;
  }
  return 0;
}

// stack frames chain_nested<murmur3> needs for a column: one per STRUCT level and per nullable LIST level, one leaf
static int frames_murmur(const srj_column& c)
{
  if (c.type_id == SRJ_LIST) return (c.null_mask ? 1 : 0) + (c.num_children > 0 ? frames_murmur(c.children[0]) : 0);
  if (c.type_id == SRJ_STRUCT) {
    int m = 0;
    for (int i = 0; i < c.num_children; ++i) m = std::max(m, frames_murmur(c.children[i]));
    return 1 + m;
  }
  return 1;
}

static int flatten(int kind, const srj_column& c, bool under_list, std::vector<HNode>& nodes, int self)
{
  HNode n{};
  n.data    = static_cast<const uint8_t*>(c.data);
  n.mask    = c.null_mask;
  n.offsets = c.offsets;
  n.type    = c.type_id;
  n.size    = type_width(c.type_id);   // STRING, LIST, STRUCT: 0
  if (n.size == 0 && c.type_id != SRJ_STRING && c.type_id != SRJ_LIST && c.type_id != SRJ_STRUCT) { set_error("hash: unsupported type id %d inside a nested column", c.type_id); return SRJ_EUNSUPPORTED; }
  if (c.type_id == SRJ_LIST) {
    if (c.num_children != 1 || !c.children || !c.offsets) { set_error("hash: a LIST column needs offsets and one child"); return SRJ_EINVAL; }
    if (kind == SRJ_HASH_MURMUR3_32 && c.children[0].type_id == SRJ_STRUCT) {
      set_error("Cannot compute hash of a table with a LIST of STRUCT columns.");   // murmur_hash.cu:173-175
      return SRJ_EINVAL;
    }
  } else if (c.type_id == SRJ_STRUCT) {
    if (c.num_children > 0 && !c.children) { set_error("hash: a STRUCT column needs its children"); return SRJ_EINVAL; }
  } else {
    if (kind == SRJ_HASH_HIVE && !hash::hive_supported(c.type_id)) { set_error("hive_hash: unsupported type id %d (hive_hash.cu:63-66)", c.type_id); return SRJ_EUNSUPPORTED; }
    if (c.type_id == SRJ_STRING ? (c.size > 0 && !c.offsets) : (c.size > 0 && !c.data)) { set_error("hash: a leaf column has no data"); return SRJ_EINVAL; }
  }
  (void)under_list;
  const int nk   = (c.type_id == SRJ_LIST || c.type_id == SRJ_STRUCT) ? c.num_children : 0;
  n.num_children = nk;
  n.first_child  = static_cast<int32_t>(nodes.size());
  nodes[self]    = n;
  nodes.resize(nodes.size() + nk);
  for (int i = 0; i < nk; ++i) {
    const int rc = flatten(kind, c.children[i], c.type_id == SRJ_LIST, nodes, n.first_child + i);
    if (rc != SRJ_OK) return rc;
  }
  return SRJ_OK;
}

bool hash_has_nested(const srj_column* cols, int32_t num_columns)
{
  for (int c = 0; c < num_columns; ++c)
    if (cols[c].type_id == SRJ_LIST || cols[c].type_id == SRJ_STRUCT) return true;
  return false;
}

// d_scratch: hash_nested_scratch_bytes() of device memory; h_pinned: the same amount of pinned host memory; both owned by
// the caller until the stream has passed this call.
int launch_hash_nested(int kind, const srj_column* cols, int32_t num_columns, int64_t num_rows, int64_t seed, void* out,
                       void* d_scratch, void* h_pinned, size_t scratch_bytes, cudaStream_t stream)
{
  std::vector<HNode> nodes(num_columns);
  std::vector<int32_t> roots(num_columns);
  for (int c = 0; c < num_columns; ++c) {
    if (cols[c].size != num_rows) { set_error("hash: column %d has %lld rows, expected %lld", c, (long long)cols[c].size, (long long)num_rows); return SRJ_EINVAL; }
    const int d = kind == SRJ_HASH_HIVE ? depth_hive(cols[c]) : depth_xx(cols[c]);
    if (d > SRJ_MAX_STACK_DEPTH) {
      set_error("The %d-th column exceeds the maximum allowed nested depth. Current depth: %d, Maximum allowed depth: %d", c, d, SRJ_MAX_STACK_DEPTH);
      return SRJ_EINVAL;
    }
    if (kind == SRJ_HASH_MURMUR3_32 && frames_murmur(cols[c]) > kMurmurStack) {
      set_error("The %d-th column nests too many nullable LIST levels for murmur3 (%d levels, at most %d)", c, frames_murmur(cols[c]), kMurmurStack);
      return SRJ_EUNSUPPORTED;
    }
    roots[c]     = c;
    const int rc = flatten(kind, cols[c], false, nodes, c);
    if (rc != SRJ_OK) return rc;
  }
  const size_t nb = nodes.size() * sizeof(HNode), rb = roots.size() * sizeof(int32_t);
  if (nb + rb + 16 > scratch_bytes) { set_error("hash: nested key tree too large (%zu nodes)", nodes.size()); return SRJ_EUNSUPPORTED; }
  std::memcpy(h_pinned, nodes.data(), nb);
  std::memcpy(static_cast<uint8_t*>(h_pinned) + nb, roots.data(), rb);
  SRJ_CUDA_TRY(cudaMemcpyAsync(d_scratch, h_pinned, nb + rb, cudaMemcpyHostToDevice, stream));
  const HNode* d_nodes   = static_cast<const HNode*>(d_scratch);
  const int32_t* d_roots = reinterpret_cast<const int32_t*>(static_cast<const uint8_t*>(d_scratch) + nb);
  const unsigned grid    = static_cast<unsigned>((num_rows + 255) / 256);
  if (kind == SRJ_HASH_XXHASH64)
    row_hash_nested_kernel<SRJ_HASH_XXHASH64><<<grid, 256, 0, stream>>>(d_nodes, d_roots, num_columns, num_rows, seed, out);
  else if (kind == SRJ_HASH_MURMUR3_32)
    row_hash_nested_kernel<SRJ_HASH_MURMUR3_32><<<grid, 256, 0, stream>>>(d_nodes, d_roots, num_columns, num_rows, seed, out);
  else
    row_hash_nested_kernel<SRJ_HASH_HIVE><<<grid, 256, 0, stream>>>(d_nodes, d_roots, num_columns, num_rows, seed, out);
  SRJ_CUDA_TRY(cudaGetLastError());
  return SRJ_OK;
}

}  // namespace srj
