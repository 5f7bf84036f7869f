// Device-resident detection post-processing for one task head, whole batch, fixed shapes.
//
// Replaces the per-sample Python loop of MultiGroupHead.get_task_detections
// (det3d/models/bbox_heads/mg_head.py:805-1085, use_multi_class_nms=False branch):
//   sigmoid scores -> score filter -> top-`nms_pre_max_size` -> anchor decode
//   (det3d/core/bbox/box_torch_ops.py:80-148) -> rotated NMS (-> csrc/nms.cu) ->
//   direction fix -> post_center_limit_range mask,
// as six launches over fixed-size buffers:
//   P1 head_scores     label (first class with the maximal fp32 score) and its logit per anchor, straight from the
//                      (possibly strided) head rows
//   P2 topk            histogram of the leading key bits (built inside P1) -> partition kernel appends the pivot
//                      bin and everything above it to a candidate list -> one CTA per sample sorts the list
//                      (value desc, index asc) in shared memory and emits the first k
//   P3 decode_selected sigmoid of the k selected anchors, compaction of those with score >= threshold (n_valid),
//                      decode of those only (the reference decodes all 70,400), direction label
//   -- d3b_rotate_nms / d3b_normal_nms on the n_valid candidates (n_valid read on the device) --
//   P4 finalize        gather the kept boxes, direction flip, range mask -> packed [B, post, nd+3] rows
// Selection matches the reference's "filter, then top-k" because sigmoid is nondecreasing: the passing anchors are the
// ones with the highest logits.  P3 still tests every selected candidate against the threshold instead of assuming a
// prefix, so the set entering NMS is exactly {score >= threshold} even where the rounding of expf is not monotonic.
// Ties in the logit go to the lower anchor index; -0 counts as +0; an anchor with a NaN logit in any class ranks
// below all others and never passes a positive threshold.
#include <algorithm>

#include "common.cuh"

namespace d3b {

constexpr int kTopkThreads = 1024;
constexpr int kTopkMax = 2048;

__device__ __forceinline__ unsigned int float_to_ordered(float f) {
  const unsigned int u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);   // ascending order as unsigned
}

// ---- P1 -------------------------------------------------------------------------------------
// grid = (CTAs per sample, batch).  Besides the best logit / label per anchor, every CTA builds a histogram of
// the top kTopkBinBits bits of the order-preserving key in shared memory and adds its non-empty bins to the
// sample's global histogram: the first radix-select pass of P2 at full-GPU width.
constexpr int kTopkBinBits = 11;
constexpr int kTopkBins = 1 << kTopkBinBits;

// torch.sigmoid in fp32: the same expression wherever a score is compared or stored
__device__ __forceinline__ float sigmoid_rn(float x) { return __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-x))); }

// The key of an anchor whose logits hold a NaN: a negative NaN whose ordered key is 0, below every other value
// (-inf included), so it is selected only when fewer than k other anchors exist and never passes a threshold.
constexpr unsigned int kNanKeyBits = 0xffffffffu;

__global__ void __launch_bounds__(256)
head_scores_kernel(const float* __restrict__ cls, int row_stride, int col0, int hw, int na, int n_cls,
                   float* __restrict__ best_logit, unsigned char* __restrict__ best_label,
                   unsigned int* __restrict__ hist) {
  __shared__ unsigned int s_hist[kTopkBins];
  const int A = hw * na, b = blockIdx.y;
  for (int j = threadIdx.x; j < kTopkBins; j += blockDim.x) s_hist[j] = 0u;
  __syncthreads();
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < A; i += gridDim.x * blockDim.x) {
    const int cell = i / na, a = i - cell * na;
    const float* p = cls + ((size_t)b * hw + cell) * row_stride + col0 + a * n_cls;
    // mg_head.py:993: torch.max over the fp32 sigmoid SCORES, first maximum wins.  Distinct logits can share a score
    // (both 1.0f once saturated), so the label is chosen on the scores; the key is the chosen class's logit, whose
    // score is the top score.  A NaN anywhere makes torch.max return NaN, which never passes `>= threshold`.
    float best = p[0];
    bool nan = isnan(best);
    int lab = 0;
    if (n_cls > 1) {
      float best_s = sigmoid_rn(best);
      for (int c = 1; c < n_cls; ++c) {
        const float v = p[c];
        nan |= isnan(v);
        const float s = sigmoid_rn(v);
        if (s > best_s) { best_s = s; best = v; lab = c; }
      }
    }
    // -0 and +0 are one logit: without this every +0 would outrank every -0 in the ordered key, whatever the index
    best = nan ? __uint_as_float(kNanKeyBits) : __fadd_rn(best, 0.0f);
    best_logit[(size_t)b * A + i] = best;
    best_label[(size_t)b * A + i] = (unsigned char)lab;
    atomicAdd(&s_hist[float_to_ordered(best) >> (32 - kTopkBinBits)], 1u);
  }
  __syncthreads();
  for (int j = threadIdx.x; j < kTopkBins; j += blockDim.x) {
    const unsigned int c = s_hist[j];
    if (c != 0u) atomicAdd(&hist[(size_t)b * kTopkBins + j], c);
  }
}

// ---- P2 -------------------------------------------------------------------------------------
// Selection order everywhere: (logit descending, anchor index ascending) -- expressed as one unique 64-bit
// composite  key << 32 | (0xffffffff - index)  sorted descending, so ties need no special handling.
__device__ __forceinline__ unsigned long long topk_composite(float v, int index) {
  return ((unsigned long long)float_to_ordered(v) << 32) | (unsigned long long)(0xffffffffu - (unsigned int)index);
}

// P2a, grid = (CTAs per sample, batch): find the pivot bin (the highest bin p with count(bin >= p) >= k) from the
// sample's histogram and append every anchor in a bin >= p to the sample's candidate list (warp-aggregated).
// The list holds the k winners plus the rest of the pivot bin -- typically k + a few hundred entries.
__global__ void __launch_bounds__(256)
topk_partition_kernel(const float* __restrict__ values, const unsigned int* __restrict__ hist, int A, int k,
                      unsigned long long* __restrict__ part, int* __restrict__ part_count) {
  __shared__ unsigned int s_group[256];
  __shared__ int s_g, s_pivot;
  __shared__ unsigned int s_acc;
  const int b = blockIdx.y, tid = threadIdx.x, lane = tid & 31;
  constexpr int kPer = kTopkBins / 256;
  unsigned int local[kPer], sum = 0u;
#pragma unroll
  for (int j = 0; j < kPer; ++j) { local[j] = hist[(size_t)b * kTopkBins + tid * kPer + j]; sum += local[j]; }
  s_group[tid] = sum;
  if (tid == 0) { s_g = 0; s_acc = 0u; s_pivot = 0; }
  __syncthreads();
  if (tid == 0) {
    unsigned int acc = 0u;
    for (int g = 255; g >= 0; --g) {
      if (acc + s_group[g] >= (unsigned int)k) { s_g = g; s_acc = acc; break; }
      acc += s_group[g];
    }
  }
  __syncthreads();
  if (tid == s_g) {
    unsigned int acc = s_acc;
    int pivot = tid * kPer;
#pragma unroll
    for (int j = kPer - 1; j >= 0; --j) {
      acc += local[j];
      if (acc >= (unsigned int)k) { pivot = tid * kPer + j; break; }
    }
    s_pivot = pivot;
  }
  __syncthreads();
  const unsigned int pivot = (unsigned int)s_pivot;
  const float* v = values + (size_t)b * A;
  unsigned long long* out = part + (size_t)b * A;
  const int a_pad = (A + 31) / 32 * 32;
  for (int i = blockIdx.x * blockDim.x + tid; i < a_pad; i += gridDim.x * blockDim.x) {
    const float x = i < A ? v[i] : 0.f;
    const bool take = i < A && (float_to_ordered(x) >> (32 - kTopkBinBits)) >= pivot;
    const unsigned int bal = __ballot_sync(0xffffffffu, take);
    if (bal == 0u) continue;
    int base = 0;
    if (lane == 0) base = atomicAdd(&part_count[b], __popc(bal));
    base = __shfl_sync(0xffffffffu, base, 0);
    if (take) out[base + __popc(bal & ((1u << lane) - 1u))] = topk_composite(x, i);
  }
}

// P2b, kTopkFinishCtas CTAs per sample: stage the candidate list in shared memory, rank it by counting and emit the
// first k in order.  A list longer than kTopkSortCap (a huge pivot bin, e.g. constant logits) is first cut down to
// exactly k entries by a radix select over the composites (unique, so the k-th largest is a strict threshold) -- one
// CTA does that sample.
constexpr int kTopkSortCap = 8192;
constexpr int kTopkFinishCtas = 16;    // CTAs per sample sharing the ranking of the candidate list

__global__ void __launch_bounds__(kTopkThreads)
topk_finish_kernel(const unsigned long long* __restrict__ part, const int* __restrict__ part_count, int A, int k,
                   float* __restrict__ out_val, int* __restrict__ out_idx) {
  extern __shared__ __align__(16) unsigned long long buf[];    // [kTopkSortCap]
  __shared__ unsigned int hist[kTopkBins];
  __shared__ unsigned long long s_prefix;
  __shared__ unsigned int s_remaining;
  __shared__ int s_count;
  const int b = blockIdx.y, tid = threadIdx.x;
  const unsigned long long* list = part + (size_t)b * A;
  const int n = min(part_count[b], A);
  int m = n;
  int cta = blockIdx.x, n_cta = gridDim.x;       // every CTA of the sample stages the whole list and ranks its share
  if (n > kTopkSortCap) {                        // (rare) radix select first: one CTA does the sample
    if (blockIdx.x != 0) return;
    cta = 0; n_cta = 1;
  }
  if (n <= kTopkSortCap) {
    for (int j = tid; j < n; j += kTopkThreads) buf[j] = list[j];
  } else {
    if (tid == 0) { s_prefix = 0ull; s_remaining = (unsigned int)k; }
    __syncthreads();
    int consumed = 0;
    while (consumed < 64) {
      const int bits = min(kTopkBinBits, 64 - consumed);
      const int shift = 64 - consumed - bits;
      for (int j = tid; j < kTopkBins; j += kTopkThreads) hist[j] = 0u;
      __syncthreads();
      const unsigned long long prefix = s_prefix;
      const int n_pad = (n + kTopkThreads - 1) / kTopkThreads * kTopkThreads;
      for (int j = tid; j < n_pad; j += kTopkThreads) {
        // this path only runs when the keys are (nearly) all equal in their leading bits, i.e. a warp's digits are
        // usually identical: one aggregated add per warp then, per-lane adds when they differ
        bool part = false;
        unsigned int digit = 0u;
        if (j < n) {
          const unsigned long long c = list[j];
          part = consumed == 0 || (c >> (64 - consumed)) == (prefix >> (64 - consumed));
          digit = (unsigned int)(c >> shift) & ((1u << bits) - 1u);
        }
        const unsigned int pm = __ballot_sync(0xffffffffu, part);
        if (pm == 0u) continue;
        const int leader = __ffs(pm) - 1;
        const unsigned int d0 = __shfl_sync(0xffffffffu, digit, leader);
        if (__all_sync(0xffffffffu, !part || digit == d0)) {
          if ((tid & 31) == leader) atomicAdd(&hist[d0], (unsigned int)__popc(pm));
        } else if (part) {
          atomicAdd(&hist[digit], 1u);
        }
      }
      __syncthreads();
      if (tid == 0) {
        unsigned int rem = s_remaining;
        int d = (1 << bits) - 1;
        for (;; --d) {
          const unsigned int c = hist[d];
          if (c >= rem || d == 0) break;
          rem -= c;
        }
        s_prefix = prefix | ((unsigned long long)d << shift);
        s_remaining = rem;
      }
      __syncthreads();
      consumed += bits;
    }
    const unsigned long long pivot = s_prefix;               // the k-th largest composite
    if (tid == 0) s_count = 0;
    __syncthreads();
    for (int j = tid; j < n; j += kTopkThreads) {
      const unsigned long long c = list[j];
      if (c >= pivot) {
        const int pos = atomicAdd(&s_count, 1);
        if (pos < kTopkSortCap) buf[pos] = c;
      }
    }
    __syncthreads();
    m = min(s_count, kTopkSortCap);
  }
  float* ov = out_val + (size_t)b * k;
  int* oi = out_idx + (size_t)b * k;
  auto emit = [&](int j, unsigned long long c) {
    const unsigned int key = (unsigned int)(c >> 32);
    const unsigned int u = (key & 0x80000000u) ? (key & 0x7fffffffu) : ~key;
    ov[j] = __uint_as_float(u);
    oi[j] = (int)(0xffffffffu - (unsigned int)c);
  };
  // Rank by counting.  The composites are unique, so the number of larger candidates IS the position in the sorted
  // order: one broadcast shared-memory read per comparison, no barriers, and the candidates spread over the sample's
  // CTAs (a bitonic network over 8192 entries in one CTA cost 59 us here; 2048 entries 21 us).
  __syncthreads();
  // A group of 32 candidates (one per lane) is ranked by the whole CTA: warp w counts over the w-th 1/32 of the list, every
  // lane of a warp reads the SAME entries (one broadcast wavefront per 16-byte read -- the loop is shared-memory-bandwidth
  // bound: splitting the list over lanes instead cost 4 wavefronts per read and measured 56 us), the 32 partial ranks per
  // candidate meet in shared memory.  Groups are dealt round-robin to the sample's CTAs.
  __shared__ int s_rank[32];
  const int warp = tid >> 5, lane = tid & 31;
  const int n_groups = (m + 31) / 32;
  const int chunk = (((m + 31) / 32) + 1) & ~1;                  // even, so the 16-byte reads stay aligned
  const int j_lo = min(warp * chunk, m), j_hi = min(j_lo + chunk, m);
  for (int g = cta; g < n_groups; g += n_cta) {                 // CTA-uniform trip count
    if (tid < 32) s_rank[tid] = 0;
    __syncthreads();
    const int c = g * 32 + lane;
    const unsigned long long x = c < m ? buf[c] : ~0ull;
    int rank = 0;
    int j = j_lo;
#pragma unroll 4
    for (; j + 2 <= j_hi; j += 2) {
      const ulonglong2 y = *reinterpret_cast<const ulonglong2*>(buf + j);
      rank += (y.x > x ? 1 : 0) + (y.y > x ? 1 : 0);
    }
    if (j < j_hi) rank += buf[j] > x ? 1 : 0;
    if (rank) atomicAdd(&s_rank[lane], rank);
    __syncthreads();
    if (warp == 0 && c < m) {
      const int r = s_rank[lane];
      if (r < k) emit(r, x);
    }
    __syncthreads();                                            // s_rank is reset by the next group
  }
  for (int j = m + cta * kTopkThreads + tid; j < k; j += n_cta * kTopkThreads) emit(j, 0ull);   // fewer candidates than k
}

// ---- P3 -------------------------------------------------------------------------------------
struct PredictDev {
  const float* box; int box_stride, box_col0;
  const float* dir; int dir_stride, dir_col0;
  const float* anchors;
  const unsigned char* best_label;
  int batch, hw, na, code, nd, k, post;
  int vec_encode, smooth_dim, norm_velo, use_rotate;
  float score_thr, direction_offset;
  float range[6];
  int has_range, label_offset;
};

// grid = (chunks of kDecodeThreads candidates, batch).  The candidates arrive in selection order; those whose score
// passes the threshold are compacted, in that order, to the front of the sample's slots (n_valid of them), and only
// they are decoded.  The passing set is exactly {score >= threshold} even where fp32 sigmoid is not monotonic in the
// logit, so it need not be a prefix of the selection.  A CTA finds its chunk's first slot by testing the chunks before
// it (one sigmoid per candidate, <= 7 rounds at k = 2048), so the decode stays spread over the SMs at batch 1.
constexpr int kDecodeThreads = 256;

__device__ __forceinline__ bool candidate_passes(const PredictDev& p, const float* sel_logit, int b, int j, float* sc) {
  const float s = sigmoid_rn(sel_logit[(size_t)b * p.k + j]);
  if (sc) *sc = s;
  return !(p.score_thr > 0.0f) || s >= p.score_thr;
}

__global__ void __launch_bounds__(kDecodeThreads)
decode_selected_kernel(PredictDev p, const float* __restrict__ sel_logit, const int* __restrict__ sel_idx,
                       float* __restrict__ cand, float* __restrict__ nms_boxes, float* __restrict__ scores,
                       int* __restrict__ labels, int* __restrict__ dir_labels, int* __restrict__ n_valid) {
  __shared__ int s_warp[kDecodeThreads / 32];
  const int A = p.hw * p.na;
  const int b = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int base = 0;
  for (int r = 0; r < (int)blockIdx.x; ++r)                     // every candidate of these chunks exists (j < k)
    base += __syncthreads_count(candidate_passes(p, sel_logit, b, r * kDecodeThreads + tid, nullptr));
  const int j = blockIdx.x * kDecodeThreads + tid;
  float sc = 0.0f;
  const bool pass = j < p.k && candidate_passes(p, sel_logit, b, j, &sc);
  const unsigned int bal = __ballot_sync(0xffffffffu, pass);
  if (lane == 0) s_warp[warp] = __popc(bal);
  __syncthreads();
  int before = 0, total = 0;
  for (int w = 0; w < kDecodeThreads / 32; ++w) {               // broadcast reads
    const int c = s_warp[w];
    before += w < warp ? c : 0;
    total += c;
  }
  if (tid == 0 && blockIdx.x == gridDim.x - 1) n_valid[b] = base + total;
  if (pass) {
    const int e = b * p.k + base + before + __popc(bal & ((1u << lane) - 1u));
    const int i = sel_idx[(size_t)b * p.k + j];
    const int cell = i / p.na, a = i - cell * p.na;
    const float* t = p.box + ((size_t)b * p.hw + cell) * p.box_stride + p.box_col0 + a * p.code;
    const float* an = p.anchors + (size_t)i * p.nd;
    // box_torch_ops.py:80-148
    const float xa = an[0], ya = an[1], za = an[2], wa = an[3], la = an[4], ha = an[5], ra = an[p.nd - 1];
    // same fp32 op sequence as the torch expression tree (separate mul / add kernels: no FMA contraction)
    const float diagonal = sqrtf(__fadd_rn(__fmul_rn(la, la), __fmul_rn(wa, wa)));
    float* o = cand + (size_t)e * p.nd;
    const float xg = __fadd_rn(__fmul_rn(t[0], diagonal), xa);
    const float yg = __fadd_rn(__fmul_rn(t[1], diagonal), ya);
    const float zg = __fadd_rn(__fmul_rn(t[2], ha), za);
    float wg, lg, hg;
    if (p.smooth_dim) {
      lg = __fmul_rn(__fadd_rn(t[4], 1.0f), la); wg = __fmul_rn(__fadd_rn(t[3], 1.0f), wa); hg = __fmul_rn(__fadd_rn(t[5], 1.0f), ha);
    } else {
      lg = __fmul_rn(expf(t[4]), la); wg = __fmul_rn(expf(t[3]), wa); hg = __fmul_rn(expf(t[5]), ha);
    }
    o[0] = xg; o[1] = yg; o[2] = zg; o[3] = wg; o[4] = lg; o[5] = hg;
    int q = 6;
    if (p.nd == 9) {
      const float vxa = an[6], vya = an[7];
      if (p.norm_velo) { o[6] = __fadd_rn(__fmul_rn(t[6], diagonal), vxa); o[7] = __fadd_rn(__fmul_rn(t[7], diagonal), vya); }
      else { o[6] = __fadd_rn(t[6], vxa); o[7] = __fadd_rn(t[7], vya); }
      q = 8;
    }
    float rg;
    if (p.vec_encode) rg = atan2f(__fadd_rn(t[q + 1], sinf(ra)), __fadd_rn(t[q], cosf(ra)));
    else rg = __fadd_rn(t[q], ra);
    o[p.nd - 1] = rg;
    float* nb = nms_boxes + (size_t)e * 5;
    if (p.use_rotate) {
      nb[0] = xg; nb[1] = yg; nb[2] = wg; nb[3] = lg; nb[4] = rg;      // mg_head.py:1008
    } else {
      // center_to_corner_box2d + corner_to_standup_nd (box_torch_ops / box_np_ops.py:267-340,419-497)
      const float s = sinf(rg), c = cosf(rg);
      const float ox[4] = {-0.5f, -0.5f, 0.5f, 0.5f}, oy[4] = {-0.5f, 0.5f, 0.5f, -0.5f};
      float mnx = 1e30f, mny = 1e30f, mxx = -1e30f, mxy = -1e30f;
      for (int c4 = 0; c4 < 4; ++c4) {
        const float px = wg * ox[c4], py = lg * oy[c4];
        const float cx = px * c + py * s + xg, cy = -px * s + py * c + yg;
        mnx = fminf(mnx, cx); mxx = fmaxf(mxx, cx); mny = fminf(mny, cy); mxy = fmaxf(mxy, cy);
      }
      nb[0] = mnx; nb[1] = mny; nb[2] = mxx; nb[3] = mxy; nb[4] = 0.0f;
    }
    scores[e] = sc;
    labels[e] = (int)p.best_label[(size_t)b * A + i] + p.label_offset;
    if (p.dir != nullptr) {
      const float* d = p.dir + ((size_t)b * p.hw + cell) * p.dir_stride + p.dir_col0 + a * 2;
      dir_labels[e] = d[1] > d[0] ? 1 : 0;                            // torch.max: first maximum wins
    }
  }
}

// ---- P4 -------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
finalize_kernel(PredictDev p, const float* __restrict__ cand, const float* __restrict__ scores,
                const int* __restrict__ labels, const int* __restrict__ dir_labels,
                const long long* __restrict__ keep_idx, const int* __restrict__ keep_count,
                float* __restrict__ packed, int packed_stride /* rows per sample in `packed` */, int row_offset) {
  const int total = p.batch * p.post;
  const int width = p.nd + 3;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < total; e += gridDim.x * blockDim.x) {
    const int b = e / p.post, j = e - b * p.post;
    float* o = packed + ((size_t)b * packed_stride + row_offset + j) * width;
    const bool have = j < keep_count[b];
    if (!have) {
      for (int c = 0; c < width; ++c) o[c] = 0.0f;
      continue;
    }
    const int src = b * p.k + (int)keep_idx[(size_t)b * p.post + j];
    const float* bx = cand + (size_t)src * p.nd;
    for (int c = 0; c < p.nd; ++c) o[c] = bx[c];
    if (p.dir != nullptr) {
      const bool opp = ((bx[p.nd - 1] - p.direction_offset) > 0.0f) != (dir_labels[src] != 0);   // mg_head.py:1044-1051
      // the reference adds torch.where(opp, pi, 0) to every angle: an angle of -0 comes out +0 when not flipped
      o[p.nd - 1] = __fadd_rn(bx[p.nd - 1], opp ? 3.14159265358979323846f : 0.0f);
    }
    bool ok = true;
    if (p.has_range) {
      for (int c = 0; c < 3; ++c) ok = ok && (o[c] >= p.range[c]) && (o[c] <= p.range[3 + c]);     // :1055-1063
    }
    o[p.nd] = scores[src];
    o[p.nd + 1] = (float)labels[src];
    o[p.nd + 2] = ok ? 1.0f : 0.0f;
  }
}

struct PredictWs {
  float* best_logit; unsigned char* best_label; unsigned int* hist; int* part_count; unsigned long long* part;
  float* sel_logit; int* sel_idx; float* cand; float* nms_boxes;
  float* scores; int* labels; int* dir_labels; int* n_valid; long long* keep_idx; int* keep_count; char* nms_ws;
  size_t nms_ws_bytes, bytes;
};

static PredictWs carve_predict(const d3b_predict_params* q, char* base) {
  PredictWs w;
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off += align_up(bytes); return base ? base + o : (char*)nullptr; };
  const size_t A = (size_t)q->hw * q->na, B = q->batch, k = q->pre_max, post = q->post_max;
  w.best_logit = (float*)take(B * A * 4);
  w.best_label = (unsigned char*)take(B * A);
  w.hist = (unsigned int*)take(B * kTopkBins * 4 + B * 4);     // histogram + list counters: one memset
  w.part_count = (int*)(w.hist ? w.hist + B * kTopkBins : nullptr);
  w.part = (unsigned long long*)take(B * A * 8);
  w.sel_logit = (float*)take(B * k * 4);
  w.sel_idx = (int*)take(B * k * 4);
  w.cand = (float*)take(B * k * q->nd * 4);
  w.nms_boxes = (float*)take(B * k * 5 * 4);
  w.scores = (float*)take(B * k * 4);
  w.labels = (int*)take(B * k * 4);
  w.dir_labels = (int*)take(B * k * 4);
  w.n_valid = (int*)take(B * 4);
  w.keep_idx = (long long*)take(B * post * 8);
  w.keep_count = (int*)take(B * 4);
  w.nms_ws_bytes = d3b_nms_workspace_bytes((int32_t)k) * (size_t)q->batch;
  w.nms_ws = take(w.nms_ws_bytes);
  w.bytes = off;
  return w;
}

}  // namespace d3b

using namespace d3b;

static int check_predict(const d3b_predict_params* q) {
  D3B_REQUIRE(q && q->cls && q->box && q->anchors, "d3b_predict_task: null argument");
  D3B_REQUIRE(q->batch >= 1 && q->hw >= 1 && q->na >= 1 && q->n_cls >= 1 && q->n_cls <= 255,
              "d3b_predict_task: bad head shape");
  D3B_REQUIRE(q->nd == 7 || q->nd == 9, "d3b_predict_task: boxes must have 7 or 9 values, got %d", q->nd);
  D3B_REQUIRE(q->code == q->nd + (q->vec_encode ? 1 : 0), "d3b_predict_task: code size %d does not match nd %d", q->code, q->nd);
  D3B_REQUIRE(q->pre_max >= 1 && q->pre_max <= kTopkMax && q->pre_max <= q->hw * q->na,
              "d3b_predict_task: nms_pre_max_size %d outside [1, min(%d, anchors)]", q->pre_max, kTopkMax);
  D3B_REQUIRE(q->post_max >= 1 && q->post_max <= q->pre_max, "d3b_predict_task: bad nms_post_max_size");
  return D3B_OK;
}

extern "C" size_t d3b_predict_workspace_bytes(const d3b_predict_params* q) {
  if (!q || q->batch < 1 || q->hw < 1 || q->na < 1 || q->pre_max < 1 || q->post_max < 1) return 0;
  return carve_predict(q, nullptr).bytes;
}

extern "C" int d3b_predict_task(const d3b_predict_params* q, float* packed, int32_t packed_rows_per_sample,
                                int32_t row_offset, int32_t* keep_counts, void* workspace, size_t workspace_bytes,
                                void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  int st = check_predict(q);
  if (st != D3B_OK) return st;
  D3B_REQUIRE(packed && workspace, "d3b_predict_task: null output/workspace");
  D3B_REQUIRE(row_offset >= 0 && row_offset + q->post_max <= packed_rows_per_sample, "d3b_predict_task: packed rows overflow");
  PredictWs w = carve_predict(q, (char*)workspace);
  if (w.bytes > workspace_bytes) {
    set_error("d3b_predict_task: workspace %zu < %zu", workspace_bytes, w.bytes);
    return D3B_ERR_WORKSPACE;
  }
  const int A = q->hw * q->na;
  PredictDev p;
  p.box = q->box; p.box_stride = q->box_row_stride; p.box_col0 = q->box_col0;
  p.dir = q->dir; p.dir_stride = q->dir_row_stride; p.dir_col0 = q->dir_col0;
  p.anchors = q->anchors; p.best_label = w.best_label;
  p.batch = q->batch; p.hw = q->hw; p.na = q->na; p.code = q->code; p.nd = q->nd; p.k = q->pre_max; p.post = q->post_max;
  p.vec_encode = q->vec_encode; p.smooth_dim = q->smooth_dim; p.norm_velo = q->norm_velo; p.use_rotate = q->use_rotate_nms;
  p.score_thr = q->score_threshold; p.direction_offset = q->direction_offset;
  for (int c = 0; c < 6; ++c) p.range[c] = q->post_center_range[c];
  p.has_range = q->has_range; p.label_offset = q->label_offset;

  static SmemOptIn finish_optin;
  D3B_CUDA(ensure_dynamic_smem(topk_finish_kernel, (size_t)kTopkSortCap * 8, finish_optin));
  D3B_CUDA(cudaMemsetAsync(w.hist, 0, (size_t)q->batch * (kTopkBins + 1) * 4, stream));
  const dim3 sample_grid((unsigned)std::min(div_up(A, 512), kNumSMs), (unsigned)q->batch);
  head_scores_kernel<<<sample_grid, 256, 0, stream>>>(q->cls, q->cls_row_stride, q->cls_col0, q->hw, q->na, q->n_cls,
                                                      w.best_logit, w.best_label, w.hist);
  D3B_LAUNCH_CHECK();
  topk_partition_kernel<<<sample_grid, 256, 0, stream>>>(w.best_logit, w.hist, A, q->pre_max, w.part, w.part_count);
  D3B_LAUNCH_CHECK();
  topk_finish_kernel<<<dim3(kTopkFinishCtas, q->batch), kTopkThreads, kTopkSortCap * 8, stream>>>(w.part, w.part_count, A, q->pre_max,
                                                                          w.sel_logit, w.sel_idx);
  D3B_LAUNCH_CHECK();
  decode_selected_kernel<<<dim3((unsigned)div_up(q->pre_max, kDecodeThreads), (unsigned)q->batch), kDecodeThreads, 0, stream>>>(
      p, w.sel_logit, w.sel_idx, w.cand, w.nms_boxes, w.scores, w.labels, w.dir_labels, w.n_valid);
  D3B_LAUNCH_CHECK();
  // one NMS per sample, all samples in the same two launches (mask, sweep)
  st = nms_batched(q->use_rotate_nms ? 1 /* xywlr, rotate_nms_cc */ : 3 /* box_torch_ops.nms "+1", mg_head.py:1013-1017 */,
                   w.nms_boxes, q->pre_max, w.n_valid, q->nms_iou_threshold, q->post_max, w.keep_idx, w.keep_count, w.nms_ws,
                   w.nms_ws_bytes, q->batch, stream);
  if (st != D3B_OK) return st;
  finalize_kernel<<<grid_for((long long)q->batch * q->post_max, 128), 128, 0, stream>>>(
      p, w.cand, w.scores, w.labels, w.dir_labels, w.keep_idx, w.keep_count, packed, packed_rows_per_sample,
      row_offset);
  D3B_LAUNCH_CHECK();
  if (keep_counts) D3B_CUDA(cudaMemcpyAsync(keep_counts, w.keep_count, (size_t)q->batch * 4, cudaMemcpyDeviceToDevice, stream));
  return D3B_OK;
}
