// k-means (k-means++ seeding + Lloyd) of one small float32 embedding, n_init restarts at once, for the spectral
// clustering of the token maps (utils/attention_utils.py:262-265 -> sklearn KMeans inside SpectralClustering).
//
// The algorithm is scikit-learn's dense KMeans.fit step for step (sklearn/cluster/_kmeans.py: KMeans.fit,
// _kmeans_plusplus, _kmeans_single_lloyd, _tolerance; _k_means_lloyd.pyx / _k_means_common.pyx: the chunked E/M step,
// _relocate_empty_clusters_dense, _average_centers, _center_shift), with the random draws taken by the host from the
// same NumPy RandomState in the same order. Precision follows scikit-learn's float32 path: k-means++ distances are
// formed in float64 (its upcast path) and stored as float32, the cumulative sum that candidates are sampled from is a
// sequential float32 sum, Lloyd distances are ||c||^2 - 2 x.c in float32. Sums scikit-learn leaves to BLAS or to a
// thread-order-dependent merge (potentials, cluster sums, inertia) are accumulated in float64 in a fixed order and
// rounded once, so the kernel is deterministic.
//
// One CTA per restart; X (centred), the running distances, the labels and the centres live in shared memory.
#include "rtti_internal.h"

#include <math.h>

namespace rtti {

constexpr int KM_THREADS = 512;
constexpr int KM_WARPS = KM_THREADS / 32;
constexpr int KM_MAX_K = 32;
constexpr int KM_MAX_N = 4096;
constexpr int KM_MAX_TRIALS = 5;   // 2 + floor(ln 32)
constexpr int KM_MAX_SMEM = 227 * 1024;   // opt-in shared memory per block on sm_90
constexpr int KM_FLAG_RELOCATION_ORDER = 1;

struct KmParams {
  const float* x;         // [n, k] row-major
  const double* draws;    // [n_init, 1 + (k-1)*trials]
  int n, k, n_init, max_iter, trials;
  float tol;
  int* labels;            // [n_init, n]
  double* inertia;        // [n_init]
  int* n_iter;            // [n_init]
  int* flags;             // [n_init]
};

struct KmShared {
  float cen[KM_MAX_K * KM_MAX_K];      // centres used by the current E-step
  float cnew[KM_MAX_K * KM_MAX_K];     // centres after the M-step
  double sums[KM_MAX_K * (KM_MAX_K + 1)];   // per cluster: feature sums, then the count
  float cnorm[KM_MAX_K];
  float weight[KM_MAX_K];
  double red[KM_WARPS * KM_MAX_TRIALS];
  double pot_t[KM_MAX_TRIALS];
  int cand[KM_MAX_TRIALS];
  float mean[KM_MAX_K];
  float var[KM_MAX_K];
  float pot;
  float tol_abs;
  int flags;
  int best;
  int stop;
};

static size_t km_smem_bytes(int n, int k) {
  return sizeof(KmShared) + static_cast<size_t>(n) * k * sizeof(float) + 2 * static_cast<size_t>(n) * sizeof(float);
}

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Block-wide sums of cnt values per thread (cnt <= KM_MAX_TRIALS), fixed order: lanes by a butterfly, warps in order.
__device__ void block_sums(double* v, int cnt, KmShared& s, double* out) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int t = 0; t < cnt; ++t) {
    const double w = warp_sum_d(v[t]);
    if (lane == 0) s.red[warp * KM_MAX_TRIALS + t] = w;
  }
  __syncthreads();
  if (threadIdx.x < cnt) {
    double a = 0.0;
    for (int w = 0; w < KM_WARPS; ++w) a += s.red[w * KM_MAX_TRIALS + threadIdx.x];
    out[threadIdx.x] = a;
  }
  __syncthreads();
}

// Squared distance of rows a and b of X, sklearn's _euclidean_distances_upcast: float64 -2 a.b + |a|^2 + |b|^2,
// clipped at 0, stored as float32.
__device__ __forceinline__ float upcast_sqdist(const float* a, const float* b, int k) {
  double dot = 0.0, aa = 0.0, bb = 0.0;
  for (int f = 0; f < k; ++f) {
    const double av = a[f], bv = b[f];
    dot = fma(av, bv, dot);
    aa = fma(av, av, aa);
    bb = fma(bv, bv, bb);
  }
  double d = -2.0 * dot;
  d += aa;
  d += bb;
  return static_cast<float>(d > 0.0 ? d : 0.0);
}

// E-step over this thread's samples: nearest centre by ||c||^2 - 2 x.c (float32, first index on a tie).
// Returns whether any label changed.
__device__ bool assign_labels(const float* X, int* lab, const KmShared& s, int n, int k) {
  bool changed = false;
  for (int i = threadIdx.x; i < n; i += KM_THREADS) {
    const float* x = X + static_cast<size_t>(i) * k;
    int best = 0;
    float bd = 0.f;
    for (int j = 0; j < k; ++j) {
      float acc = 0.f;
      for (int f = 0; f < k; ++f) acc = fmaf(x[f], s.cen[j * k + f], acc);
      const float d = fmaf(-2.f, acc, s.cnorm[j]);
      if (j == 0 || d < bd) { bd = d; best = j; }
    }
    changed |= lab[i] != best;
    lab[i] = best;
  }
  return changed;
}

__device__ void centre_norms(KmShared& s, int k) {
  if (threadIdx.x < k) {
    float a = 0.f;
    for (int f = 0; f < k; ++f) a = __fadd_rn(a, __fmul_rn(s.cen[threadIdx.x * k + f], s.cen[threadIdx.x * k + f]));
    s.cnorm[threadIdx.x] = a;
  }
}

__global__ void __launch_bounds__(KM_THREADS, 1) kmeans_fit_kernel(const __grid_constant__ KmParams p) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  KmShared& s = *reinterpret_cast<KmShared*>(smem_raw);
  const int n = p.n, k = p.k, T = p.trials, r = blockIdx.x, tid = threadIdx.x;
  float* X = reinterpret_cast<float*>(smem_raw + sizeof(KmShared));   // [n, k], centred
  float* dist = X + static_cast<size_t>(n) * k;                        // [n] closest squared distance / scratch
  int* lab = reinterpret_cast<int*>(dist + n);                         // [n]
  const double* draws = p.draws + static_cast<size_t>(r) * (1 + (k - 1) * T);

  for (int e = tid; e < n * k; e += KM_THREADS) X[e] = p.x[e];
  for (int i = tid; i < n; i += KM_THREADS) lab[i] = -1;
  if (tid == 0) s.flags = 0;
  __syncthreads();
  // _tolerance on the input, then centring (KMeans.fit): float32 column sums in row order, as numpy's axis-0 reduction.
  if (tid < k) {
    float a = 0.f;
    for (int i = 0; i < n; ++i) a = __fadd_rn(a, X[i * k + tid]);
    const float m = __fdiv_rn(a, static_cast<float>(n));
    float v = 0.f;
    for (int i = 0; i < n; ++i) {
      const float d = __fsub_rn(X[i * k + tid], m);
      v = __fadd_rn(v, __fmul_rn(d, d));
    }
    s.mean[tid] = m;
    s.var[tid] = __fdiv_rn(v, static_cast<float>(n));
  }
  __syncthreads();
  if (tid == 0) {
    float a = 0.f;
    for (int f = 0; f < k; ++f) a = __fadd_rn(a, s.var[f]);
    s.tol_abs = __fmul_rn(__fdiv_rn(a, static_cast<float>(k)), p.tol);
  }
  for (int e = tid; e < n * k; e += KM_THREADS) X[e] = __fsub_rn(X[e], s.mean[e % k]);
  __syncthreads();

  // ---- k-means++ (_kmeans_plusplus) ----
  {
    const int c0 = static_cast<int>(draws[0]);
    double part = 0.0;
    for (int i = tid; i < n; i += KM_THREADS) {
      dist[i] = upcast_sqdist(X + static_cast<size_t>(c0) * k, X + static_cast<size_t>(i) * k, k);
      part += dist[i];
    }
    if (tid < k) s.cen[tid] = X[static_cast<size_t>(c0) * k + tid];
    double tot;
    block_sums(&part, 1, s, &tot);
    if (tid == 0) s.pot = static_cast<float>(tot);
    __syncthreads();
  }
  for (int c = 1; c < k; ++c) {
    if (tid == 0) {
      // searchsorted(cumsum(closest), u * pot, side='left') for every trial in one sequential float32 scan
      double rv[KM_MAX_TRIALS];
      int idx[KM_MAX_TRIALS];
      for (int t = 0; t < T; ++t) { rv[t] = draws[1 + (c - 1) * T + t] * static_cast<double>(s.pot); idx[t] = -1; }
      float cum = 0.f;
      int open = T;
      for (int i = 0; i < n && open > 0; ++i) {
        cum = __fadd_rn(cum, dist[i]);
        for (int t = 0; t < T; ++t)
          if (idx[t] < 0 && static_cast<double>(cum) >= rv[t]) { idx[t] = i; --open; }
      }
      for (int t = 0; t < T; ++t) s.cand[t] = idx[t] < 0 ? n - 1 : idx[t];
    }
    __syncthreads();
    double part[KM_MAX_TRIALS];
    for (int t = 0; t < T; ++t) part[t] = 0.0;
    for (int i = tid; i < n; i += KM_THREADS) {
      const float* xi = X + static_cast<size_t>(i) * k;
      for (int t = 0; t < T; ++t) part[t] += fminf(dist[i], upcast_sqdist(X + static_cast<size_t>(s.cand[t]) * k, xi, k));
    }
    block_sums(part, T, s, s.pot_t);
    if (tid == 0) {
      int b = 0;
      for (int t = 1; t < T; ++t)
        if (static_cast<float>(s.pot_t[t]) < static_cast<float>(s.pot_t[b])) b = t;
      s.best = s.cand[b];
      s.pot = static_cast<float>(s.pot_t[b]);
    }
    __syncthreads();
    const int bc = s.best;
    for (int i = tid; i < n; i += KM_THREADS)
      dist[i] = fminf(dist[i], upcast_sqdist(X + static_cast<size_t>(bc) * k, X + static_cast<size_t>(i) * k, k));
    if (tid < k) s.cen[c * k + tid] = X[static_cast<size_t>(bc) * k + tid];
    __syncthreads();
  }

  // ---- Lloyd (_kmeans_single_lloyd) ----
  const int lane = tid & 31, warp = tid >> 5;
  const int kk = k * k;
  int it = 0;
  bool strict = false;
  for (it = 0; it < p.max_iter; ++it) {
    centre_norms(s, k);
    __syncthreads();
    const bool changed = __syncthreads_or(assign_labels(X, lab, s, n, k));
    // M-step: per (cluster, feature) sums and per-cluster counts, one warp per pair, float64, fixed order
    for (int q = warp; q < k * (k + 1); q += KM_WARPS) {
      const int j = q / (k + 1), f = q % (k + 1);
      double a = 0.0;
      for (int i = lane; i < n; i += 32)
        if (lab[i] == j) a += f < k ? static_cast<double>(X[static_cast<size_t>(i) * k + f]) : 1.0;
      a = warp_sum_d(a);
      if (lane == 0) s.sums[q] = a;
    }
    __syncthreads();
    // _relocate_empty_clusters_dense: empty clusters take the samples farthest from their centre
    bool any_empty = false;
    for (int j = 0; j < k; ++j) any_empty |= s.sums[j * (k + 1) + k] == 0.0;
    if (any_empty) {
      for (int i = tid; i < n; i += KM_THREADS) {
        const float* x = X + static_cast<size_t>(i) * k;
        float a = 0.f;
        for (int f = 0; f < k; ++f) {
          const float d = __fsub_rn(x[f], s.cen[lab[i] * k + f]);
          a = __fadd_rn(a, __fmul_rn(d, d));
        }
        dist[i] = a;
      }
      __syncthreads();
      if (tid == 0) {
        float dmax = 0.f;
        for (int i = 0; i < n; ++i) dmax = fmaxf(dmax, dist[i]);
        if (dmax > 0.f) {
          // scikit-learn takes the farthest samples from np.argpartition, which leaves the order of several samples
          // (several empty clusters, or distinct samples tied at the largest distance) unspecified: flag the restart.
          int n_empty = 0;
          for (int j = 0; j < k; ++j) n_empty += s.sums[j * (k + 1) + k] == 0.0;
          if (n_empty > 1) s.flags |= KM_FLAG_RELOCATION_ORDER;
          // farthest first (first index on a tie); a chosen sample is marked with -1
          for (int j = 0; j < k; ++j) {
            if (s.sums[j * (k + 1) + k] != 0.0) continue;
            int far = 0;
            for (int i = 1; i < n; ++i)
              if (dist[i] > dist[far]) far = i;
            for (int i = far + 1; i < n; ++i) {
              if (dist[i] != dist[far]) continue;
              for (int f = 0; f < k; ++f)
                if (X[static_cast<size_t>(i) * k + f] != X[static_cast<size_t>(far) * k + f]) s.flags |= KM_FLAG_RELOCATION_ORDER;
            }
            dist[far] = -1.f;
            const int old = lab[far];
            for (int f = 0; f < k; ++f) {
              const double xv = X[static_cast<size_t>(far) * k + f];
              s.sums[old * (k + 1) + f] -= xv;
              s.sums[j * (k + 1) + f] = xv;
            }
            s.sums[j * (k + 1) + k] = 1.0;
            s.sums[old * (k + 1) + k] -= 1.0;
          }
        }
      }
      __syncthreads();
    }
    // _average_centers + _center_shift
    if (tid == 0) {
      int amax = 0;
      for (int j = 0; j < k; ++j) {
        s.weight[j] = static_cast<float>(s.sums[j * (k + 1) + k]);
        if (s.weight[j] > s.weight[amax]) amax = j;
      }
      // one pass in cluster order, as _average_centers: an empty cluster copies the heaviest cluster's centre as it
      // stands at that point (still the unscaled sum when the heaviest cluster comes later)
      for (int j = 0; j < k; ++j)
        for (int f = 0; f < k; ++f) s.cnew[j * k + f] = static_cast<float>(s.sums[j * (k + 1) + f]);
      for (int j = 0; j < k; ++j) {
        if (s.weight[j] > 0.f) {
          const float alpha = __fdiv_rn(1.f, s.weight[j]);
          for (int f = 0; f < k; ++f) s.cnew[j * k + f] = __fmul_rn(s.cnew[j * k + f], alpha);
        } else {
          for (int f = 0; f < k; ++f) s.cnew[j * k + f] = s.cnew[amax * k + f];
        }
      }
      float shift_tot = 0.f;
      for (int j = 0; j < k; ++j) {
        float a = 0.f;
        for (int f = 0; f < k; ++f) {
          const float d = __fsub_rn(s.cnew[j * k + f], s.cen[j * k + f]);
          a = __fadd_rn(a, __fmul_rn(d, d));
        }
        const float sh = __fsqrt_rn(a);
        shift_tot = __fadd_rn(shift_tot, __fmul_rn(sh, sh));
      }
      s.stop = !changed ? 2 : (shift_tot <= s.tol_abs ? 1 : 0);
    }
    __syncthreads();
    for (int e = tid; e < kk; e += KM_THREADS) s.cen[e] = s.cnew[e];
    const int stop = s.stop;
    __syncthreads();
    if (stop) {
      strict = stop == 2;
      break;
    }
  }
  if (it == p.max_iter) it = p.max_iter - 1;
  if (!strict) {   // labels must match the final centres
    centre_norms(s, k);
    __syncthreads();
    assign_labels(X, lab, s, n, k);
    __syncthreads();
  }
  // inertia of the final labels, float32 per sample, summed in float64
  double part = 0.0;
  for (int i = tid; i < n; i += KM_THREADS) {
    const float* x = X + static_cast<size_t>(i) * k;
    float a = 0.f;
    for (int f = 0; f < k; ++f) {
      const float d = __fsub_rn(x[f], s.cen[lab[i] * k + f]);
      a = __fadd_rn(a, __fmul_rn(d, d));
    }
    part += a;
    p.labels[static_cast<size_t>(r) * n + i] = lab[i];
  }
  double tot;
  block_sums(&part, 1, s, &tot);
  if (tid == 0) {
    p.inertia[r] = tot;
    p.n_iter[r] = it + 1;
    p.flags[r] = s.flags;
  }
}

}  // namespace rtti

using namespace rtti;

// n_local_trials of _kmeans_plusplus
static int km_trials(int k) { return 2 + static_cast<int>(log(static_cast<double>(k))); }

extern "C" int rtti_kmeans_supported(int n, int k) {
  if (k < 1 || k > KM_MAX_K || n < k || n > KM_MAX_N) return RTTI_ERR_SHAPE;
  return km_smem_bytes(n, k) <= static_cast<size_t>(KM_MAX_SMEM) ? RTTI_OK : RTTI_ERR_SHAPE;
}

extern "C" int rtti_kmeans_fit(const float* x, const double* draws, int n, int k, int n_init, int max_iter, double tol,
                               int* labels, double* inertia, int* n_iter, int* flags, void* stream) {
  if (!x || !draws || !labels || !inertia || !n_iter || !flags) return RTTI_ERR_ARG;
  if (n_init < 1 || max_iter < 1 || !(tol >= 0.0)) return RTTI_ERR_ARG;
  int rc = rtti_kmeans_supported(n, k);
  if (rc != RTTI_OK) return rc;
  const size_t smem = km_smem_bytes(n, k);
  rc = rtti_arch_ok();
  if (rc != RTTI_OK) return rc;
  static const bool configured = cudaFuncSetAttribute(kmeans_fit_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                      KM_MAX_SMEM) == cudaSuccess;
  if (!configured) return RTTI_ERR_CUDA;
  KmParams p{};
  p.x = x; p.draws = draws; p.n = n; p.k = k; p.n_init = n_init; p.max_iter = max_iter;
  p.trials = km_trials(k);
  p.tol = static_cast<float>(tol);
  p.labels = labels; p.inertia = inertia; p.n_iter = n_iter; p.flags = flags;
  kmeans_fit_kernel<<<n_init, KM_THREADS, smem, (cudaStream_t)stream>>>(p);
  return cudaGetLastError() == cudaSuccess ? RTTI_OK : RTTI_ERR_CUDA;
}
