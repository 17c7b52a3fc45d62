// bn.cu -- BatchNorm3d with batch statistics (training mode, freeze_stats=False) around the identity-epilogue convolution of a
// Unit3Dpy (i3dpt.py:103-111; models/networks.py:85-99, two_branch.py:146-161 leave every BatchNorm in training mode):
//   statistics  mean / biased variance of z [M, C] over the M = N*T*H*W pixels, the folded (scale, shift), and the momentum
//               update of the running statistics with the unbiased variance (torch.nn.functional.batch_norm, training=True)
//   apply       y = relu(scale * z + shift) into up to three destinations (the column ranges of the fused 1x1 branches)
//   backward    dz = gamma * rstd * (g - mean(g) - xhat * mean(g * xhat)), dgamma = sum g * xhat, dbeta = sum g  (g = dy [y > 0])
// z, y, dy and dz are channel slices (ld) of fp16 or fp32 buffers; statistics and sums are fp32.  Every reduction forms
// per-chunk partials that a second kernel combines in a fixed order: no atomics, bit-identical from run to run.
// Synchronised BatchNorm (several ranks normalising with the statistics of all their rows) runs the same kernels split in
// two: the local entries stop at each rank's merged (count, mean, M2) or raw sums, and the merge entries run the combining
// kernel over every rank's result as its chunks.
#include "common.cuh"

using namespace step;

namespace {

constexpr int kRowsPerChunk = 256, kMaxChunks = 512;

int bn_chunks(long long M) {
  const long long c = (M + kRowsPerChunk - 1) / kRowsPerChunk;
  return (int)(c < kMaxChunks ? c : kMaxChunks);
}

// Chan et al.'s merge of two (count, mean, M2) triples; an empty side leaves the other unchanged.
__device__ __forceinline__ void chan_merge(float& n, float& mean, float& m2, float nb, float meanb, float m2b) {
  if (nb == 0.0f) return;
  if (n == 0.0f) {
    n = nb; mean = meanb; m2 = m2b;
    return;
  }
  const float nn = n + nb, d = meanb - mean, f = nb / nn;
  mean += d * f;
  m2 += m2b + d * d * n * f;
  n = nn;
}

// Per-chunk (count, mean, M2) of every channel.  The block holds `cols` channel vectors of `rows` pixels (cols * rows <= 256
// threads); each thread runs Welford's update over its pixels of the chunk (ascending), then the block's rows are merged in
// ascending order.  partial: [chunks, 3, C] fp32.
template <typename T>
__global__ void __launch_bounds__(256) bn_stats_partial_kernel(const T* __restrict__ z, int z_ld, long long M, int C, int cols,
                                                               int rows, long long rows_per_chunk, float* __restrict__ partial) {
  constexpr int V = Vec16<T>::N;
  __shared__ float red_n[256], red_mean[256 * V], red_m2[256 * V];
  const int cv = C / V;
  const int t = threadIdx.x, col = t % cols, r = t / cols;
  const int cvec = blockIdx.y * cols + col;
  const int c = cvec * V;
  float n = 0.0f, mean[V], m2[V];
#pragma unroll
  for (int k = 0; k < V; ++k) mean[k] = m2[k] = 0.0f;
  if (r < rows && cvec < cv) {
    const long long m0 = (long long)blockIdx.x * rows_per_chunk, m1 = m0 + rows_per_chunk < M ? m0 + rows_per_chunk : M;
    for (long long m = m0 + r; m < m1; m += rows) {
      float v[V];
      load16(z + (size_t)m * z_ld + c, v);
      n += 1.0f;
      const float inv = 1.0f / n;
#pragma unroll
      for (int k = 0; k < V; ++k) {
        const float d = v[k] - mean[k];
        mean[k] += d * inv;
        m2[k] += d * (v[k] - mean[k]);
      }
    }
  }
  if (r < rows) {
    if (col == 0) red_n[r] = n;
#pragma unroll
    for (int k = 0; k < V; ++k) {
      red_mean[r * cols * V + col * V + k] = mean[k];
      red_m2[r * cols * V + col * V + k] = m2[k];
    }
  }
  __syncthreads();
  const int width = cols * V;
  for (int ch = t; ch < width; ch += blockDim.x) {
    const int cg = blockIdx.y * width + ch;
    if (cg >= C) continue;
    float an = 0.0f, am = 0.0f, a2 = 0.0f;
    for (int q = 0; q < rows; ++q) chan_merge(an, am, a2, red_n[q], red_mean[q * width + ch], red_m2[q * width + ch]);
    float* p = partial + (size_t)blockIdx.x * 3 * C + cg;
    p[0] = an;
    p[C] = am;
    p[2 * C] = a2;
  }
}

// The chunks merged in a fixed order, one warp per channel: lane l merges chunks l, l + 32, ... in order, then a fixed
// pairwise tree merges the lanes -> mean, rstd = 1 / sqrt(var + eps) (biased variance), scale = gamma * rstd,
// shift = beta - mean * scale; with running statistics: running = (1 - momentum) * running + momentum * batch, unbiased
// variance.  partial: [chunks, 3, ld].  With `triple` the merged (count, mean, M2) go to triple [3, triple_ld] instead and
// nothing is folded (step_bn_stats_local): the same kernel then merges every rank's triple as its chunks
// (step_bn_stats_merge), so a single rank's result is the fused entry's bit for bit.
constexpr int kFinalWarps = 8;
__global__ void __launch_bounds__(32 * kFinalWarps) bn_stats_final_kernel(const float* __restrict__ partial, int chunks, int ld, int C,
                                                                          long long M, const float* __restrict__ gamma,
                                                                          const float* __restrict__ beta, float eps, float momentum,
                                                                          float* __restrict__ running_mean,
                                                                          float* __restrict__ running_var,
                                                                          float* __restrict__ mean_out, float* __restrict__ rstd_out,
                                                                          float* __restrict__ scale, float* __restrict__ shift,
                                                                          float* __restrict__ triple, int triple_ld) {
  const int lane = threadIdx.x & 31, c = blockIdx.x * kFinalWarps + (threadIdx.x >> 5);
  if (c >= C) return;   // uniform over the warp
  float n = 0.0f, mean = 0.0f, m2 = 0.0f;
  for (int k = lane; k < chunks; k += 32) {
    const float* p = partial + (size_t)k * 3 * ld + c;
    chan_merge(n, mean, m2, p[0], p[ld], p[2 * ld]);
  }
  for (int off = 1; off < 32; off <<= 1) {
    const float nb = __shfl_down_sync(0xffffffffu, n, off), mb = __shfl_down_sync(0xffffffffu, mean, off),
                m2b = __shfl_down_sync(0xffffffffu, m2, off);
    if ((lane & (2 * off - 1)) == 0) chan_merge(n, mean, m2, nb, mb, m2b);
  }
  if (lane != 0) return;
  if (triple) {
    triple[c] = n;
    triple[triple_ld + c] = mean;
    triple[2 * triple_ld + c] = m2;
    return;
  }
  const float var = m2 / (float)M;
  const float rstd = 1.0f / sqrtf(var + eps);
  const float s = gamma[c] * rstd;
  mean_out[c] = mean;
  rstd_out[c] = rstd;
  scale[c] = s;
  shift[c] = beta[c] - mean * s;
  if (running_mean) {
    const float var_u = m2 / (float)(M - 1);
    running_mean[c] = (1.0f - momentum) * running_mean[c] + momentum * mean;
    running_var[c] = (1.0f - momentum) * running_var[c] + momentum * var_u;
  }
}

// y = relu(scale * z + shift): columns [0, split1) to y0, [split1, split2) to y1, [split2, C) to y2, each at its own column 0.
template <typename T>
__global__ void __launch_bounds__(256) bn_apply_kernel(const T* __restrict__ z, int z_ld, long long M, int C,
                                                       const float* __restrict__ scale, const float* __restrict__ shift, int relu,
                                                       T* __restrict__ y0, int y0_ld, int split1, T* __restrict__ y1, int y1_ld,
                                                       int split2, T* __restrict__ y2, int y2_ld) {
  constexpr int V = Vec16<T>::N;
  const int cv = C / V;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M * cv) return;
  const long long m = i / cv;
  const int c = (int)(i - m * cv) * V;
  float v[V];
  load16(z + (size_t)m * z_ld + c, v);
#pragma unroll
  for (int k = 0; k < V; ++k) {
    v[k] = scale[c + k] * v[k] + shift[c + k];
    if (relu) v[k] = v[k] > 0.0f ? v[k] : 0.0f;
  }
  T* dst = c < split1 ? y0 + (size_t)m * y0_ld + c
         : c < split2 ? y1 + (size_t)m * y1_ld + (c - split1)
                      : y2 + (size_t)m * y2_ld + (c - split2);
  store16(dst, v);
}

// Per-chunk partials of  sum g  and  sum g * xhat  (g = dy [y > 0], xhat = (z - mean) * rstd), laid out and added as in
// bn_stats_partial_kernel.  partial: [chunks, 2, C].
template <typename T>
__global__ void __launch_bounds__(256) bn_bwd_partial_kernel(const T* __restrict__ dy, int dy_ld, const T* __restrict__ y, int y_ld,
                                                             const T* __restrict__ z, int z_ld, long long M, int C,
                                                             const float* __restrict__ mean, const float* __restrict__ rstd,
                                                             int relu, int cols, int rows, long long rows_per_chunk,
                                                             float* __restrict__ partial) {
  constexpr int V = Vec16<T>::N;
  __shared__ float red[2][256 * V];
  const int cv = C / V;
  const int t = threadIdx.x, col = t % cols, r = t / cols;
  const int cvec = blockIdx.y * cols + col;
  const int c = cvec * V;
  float sg[V], sgx[V];
#pragma unroll
  for (int k = 0; k < V; ++k) sg[k] = sgx[k] = 0.0f;
  if (r < rows && cvec < cv) {
    float mu[V], rs[V];
#pragma unroll
    for (int k = 0; k < V; ++k) {
      mu[k] = mean[c + k];
      rs[k] = rstd[c + k];
    }
    const long long m0 = (long long)blockIdx.x * rows_per_chunk, m1 = m0 + rows_per_chunk < M ? m0 + rows_per_chunk : M;
    for (long long m = m0 + r; m < m1; m += rows) {
      float g[V], zz[V];
      load16(dy + (size_t)m * dy_ld + c, g);
      load16(z + (size_t)m * z_ld + c, zz);
      if (relu) {
        float v[V];
        load16(y + (size_t)m * y_ld + c, v);
#pragma unroll
        for (int k = 0; k < V; ++k) g[k] = v[k] > 0.0f ? g[k] : 0.0f;
      }
#pragma unroll
      for (int k = 0; k < V; ++k) {
        sg[k] += g[k];
        sgx[k] += g[k] * ((zz[k] - mu[k]) * rs[k]);
      }
    }
  }
  if (r < rows) {
#pragma unroll
    for (int k = 0; k < V; ++k) {
      red[0][r * cols * V + col * V + k] = sg[k];
      red[1][r * cols * V + col * V + k] = sgx[k];
    }
  }
  __syncthreads();
  const int width = cols * V;
  for (int j = t; j < 2 * width; j += blockDim.x) {
    const int which = j / width, ch = j - which * width;
    if (blockIdx.y * width + ch >= C) continue;
    float acc = 0.0f;
    for (int q = 0; q < rows; ++q) acc += red[which][q * width + ch];
    partial[((size_t)blockIdx.x * 2 + which) * C + blockIdx.y * width + ch] = acc;
  }
}

// Chunk sums in order (partial: [chunks, 2, ld]) -> dbeta = gscale * sum g, dgamma = gscale * sum g xhat, the raw sums to
// sums [2, sums_ld] (step_bn_bwd_sums), and the coefficients of the dz pass: coef [3, C] = (gamma * rstd, sum g / M,
// sum g xhat / M).  Every output may be NULL.  Run over every rank's raw sums as its chunks (step_bn_bwd_merge_dz) it forms
// the coefficients of the whole batch; with one rank, 0.0f + s == s (a sum from 0.0f is never -0.0f) keeps them the fused
// entry's bit for bit.
__global__ void __launch_bounds__(256) bn_bwd_reduce_kernel(const float* __restrict__ partial, int chunks, int ld, int C, long long M,
                                                            const float* __restrict__ gamma, const float* __restrict__ rstd,
                                                            float gscale, float* __restrict__ dgamma, float* __restrict__ dbeta,
                                                            float* __restrict__ sums, int sums_ld, float* __restrict__ coef) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float sg = 0.0f, sgx = 0.0f;
  for (int k = 0; k < chunks; ++k) {
    sg += partial[(size_t)k * 2 * ld + c];
    sgx += partial[((size_t)k * 2 + 1) * ld + c];
  }
  if (dbeta) dbeta[c] = sg * gscale;
  if (dgamma) dgamma[c] = sgx * gscale;
  if (sums) {
    sums[c] = sg;
    sums[sums_ld + c] = sgx;
  }
  if (!coef) return;
  coef[c] = gamma[c] * rstd[c];
  coef[C + c] = sg / (float)M;
  coef[2 * C + c] = sgx / (float)M;
}

// dz = gamma * rstd * (g - mean(g) - xhat * mean(g xhat)), in the storage type, at dz_ld.
template <typename T>
__global__ void __launch_bounds__(256) bn_bwd_dz_kernel(const T* __restrict__ dy, int dy_ld, const T* __restrict__ y, int y_ld,
                                                        const T* __restrict__ z, int z_ld, long long M, int C,
                                                        const float* __restrict__ mean, const float* __restrict__ rstd, int relu,
                                                        const float* __restrict__ coef, T* __restrict__ dz, int dz_ld) {
  constexpr int V = Vec16<T>::N;
  const int cv = C / V;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M * cv) return;
  const long long m = i / cv;
  const int c = (int)(i - m * cv) * V;
  float g[V], zz[V];
  load16(dy + (size_t)m * dy_ld + c, g);
  load16(z + (size_t)m * z_ld + c, zz);
  if (relu) {
    float v[V];
    load16(y + (size_t)m * y_ld + c, v);
#pragma unroll
    for (int k = 0; k < V; ++k) g[k] = v[k] > 0.0f ? g[k] : 0.0f;
  }
#pragma unroll
  for (int k = 0; k < V; ++k) {
    const float xhat = (zz[k] - mean[c + k]) * rstd[c + k];
    g[k] = coef[c + k] * (g[k] - coef[C + c + k] - xhat * coef[2 * C + c + k]);
  }
  store16(dz + (size_t)m * dz_ld + c, g);
}

inline bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

template <typename T>
int bn_stats_launch(const void* z, int z_ld, long long M, int C, const float* gamma, const float* beta, float eps, float momentum,
                    float* running_mean, float* running_var, float* mean, float* rstd, float* scale, float* shift, void* workspace,
                    size_t ws_bytes, step_stream_t stream) {
  constexpr int V = Vec16<T>::N;
  STEP_CHECK_ARG(z && gamma && beta && mean && rstd && scale && shift && workspace && C > 0, "bn_stats: bad arguments");
  STEP_CHECK_ARG(M > 1, "bn_stats: Expected more than 1 value per channel when training (M=%lld)", M);
  STEP_CHECK_ARG(!running_mean == !running_var, "bn_stats: give both running statistics or neither");
  STEP_CHECK_ARG(C % V == 0 && z_ld % V == 0 && z_ld >= C, "bn_stats: C and z_ld must be multiples of %d, z_ld >= C (C=%d z_ld=%d)",
                 V, C, z_ld);
  STEP_CHECK_ARG(aligned16(z), "bn_stats: z must be 16-byte aligned");
  STEP_CHECK_ARG(eps > 0.0f && momentum >= 0.0f && momentum <= 1.0f, "bn_stats: eps %g must be > 0 and momentum %g in [0, 1]",
                 eps, momentum);
  const size_t need = step_bn_stats_workspace_bytes(M, C);
  if (ws_bytes < need) return fail(STEP_E_WORKSPACE, "bn_stats: workspace %zu < %zu", ws_bytes, need);
  const int cv = C / V, cols = cv < 256 ? cv : 256, rows = 256 / cols;
  const int chunks = bn_chunks(M);
  const long long rows_per_chunk = (M + chunks - 1) / chunks;
  bn_stats_partial_kernel<T><<<dim3(chunks, ceil_div(cv, cols)), 256, 0, cu(stream)>>>((const T*)z, z_ld, M, C, cols, rows,
                                                                                        rows_per_chunk, (float*)workspace);
  STEP_LAUNCH_CHECK("bn_stats_partial_kernel");
  bn_stats_final_kernel<<<ceil_div(C, kFinalWarps), 32 * kFinalWarps, 0, cu(stream)>>>((const float*)workspace, chunks, C, C, M, gamma, beta, eps, momentum,
                                                                  running_mean, running_var, mean, rstd, scale, shift, nullptr, 0);
  STEP_LAUNCH_CHECK("bn_stats_final_kernel");
  return 0;
}

template <typename T>
int bn_apply_launch(const void* z, int z_ld, long long M, int C, const float* scale, const float* shift, int relu, void* y, int y_ld,
                    int split1, void* y1, int y1_ld, int split2, void* y2, int y2_ld, step_stream_t stream) {
  constexpr int V = Vec16<T>::N;
  STEP_CHECK_ARG(z && scale && shift && y && M > 0 && C > 0, "bn_apply: bad arguments");
  STEP_CHECK_ARG(0 < split1 && split1 <= split2 && split2 <= C && (split2 == split1 || y1) && (split2 == C || y2),
                 "bn_apply: the column ranges [0, %d) [%d, %d) [%d, %d) need a destination each", split1, split1, split2, split2, C);
  STEP_CHECK_ARG(C % V == 0 && split1 % V == 0 && split2 % V == 0 && z_ld % V == 0 && z_ld >= C && y_ld % V == 0 && y_ld >= split1 &&
                 (!y1 || (y1_ld % V == 0 && y1_ld >= split2 - split1)) && (!y2 || (y2_ld % V == 0 && y2_ld >= C - split2)),
                 "bn_apply: C, the splits and the ld arguments must be multiples of %d and each ld wide enough (C=%d z_ld=%d "
                 "y_ld=%d)", V, C, z_ld, y_ld);
  STEP_CHECK_ARG(aligned16(z) && aligned16(y) && aligned16(y1) && aligned16(y2), "bn_apply: pointers must be 16-byte aligned");
  bn_apply_kernel<T><<<ceil_div(M * (C / V), 256), 256, 0, cu(stream)>>>((const T*)z, z_ld, M, C, scale, shift, relu, (T*)y, y_ld,
                                                                         split1, (T*)y1, y1_ld, split2, (T*)y2, y2_ld);
  STEP_LAUNCH_CHECK("bn_apply_kernel");
  return 0;
}

template <typename T>
int bn_bwd_launch(const void* dy, int dy_ld, const void* y, int y_ld, const void* z, int z_ld, long long M, int C, const float* mean,
                  const float* rstd, const float* gamma, int relu, float gscale, void* dz, int dz_ld, float* dgamma, float* dbeta,
                  void* workspace, size_t ws_bytes, step_stream_t stream) {
  constexpr int V = Vec16<T>::N;
  STEP_CHECK_ARG(dy && z && dz && mean && rstd && gamma && workspace && (!relu || y) && C > 0, "bn_bwd: bad arguments");
  STEP_CHECK_ARG(M > 1, "bn_bwd: Expected more than 1 value per channel when training (M=%lld)", M);
  STEP_CHECK_ARG(C % V == 0 && dy_ld % V == 0 && z_ld % V == 0 && dz_ld % V == 0 && (!relu || y_ld % V == 0) && dy_ld >= C &&
                 z_ld >= C && dz_ld >= C && (!relu || y_ld >= C),
                 "bn_bwd: C and the ld arguments must be multiples of %d, each ld >= C (C=%d dy_ld=%d y_ld=%d z_ld=%d dz_ld=%d)", V, C,
                 dy_ld, y_ld, z_ld, dz_ld);
  STEP_CHECK_ARG(aligned16(dy) && aligned16(y) && aligned16(z) && aligned16(dz), "bn_bwd: pointers must be 16-byte aligned");
  const size_t need = step_bn_bwd_workspace_bytes(M, C);
  if (ws_bytes < need) return fail(STEP_E_WORKSPACE, "bn_bwd: workspace %zu < %zu", ws_bytes, need);
  const int cv = C / V, cols = cv < 256 ? cv : 256, rows = 256 / cols;
  const int chunks = bn_chunks(M);
  const long long rows_per_chunk = (M + chunks - 1) / chunks;
  float* partial = (float*)workspace;
  float* coef = partial + (size_t)chunks * 2 * C;
  bn_bwd_partial_kernel<T><<<dim3(chunks, ceil_div(cv, cols)), 256, 0, cu(stream)>>>(
      (const T*)dy, dy_ld, (const T*)y, y_ld, (const T*)z, z_ld, M, C, mean, rstd, relu, cols, rows, rows_per_chunk, partial);
  STEP_LAUNCH_CHECK("bn_bwd_partial_kernel");
  bn_bwd_reduce_kernel<<<ceil_div(C, 256), 256, 0, cu(stream)>>>(partial, chunks, C, C, M, gamma, rstd, gscale, dgamma, dbeta, nullptr, 0,
                                                                 coef);
  STEP_LAUNCH_CHECK("bn_bwd_reduce_kernel");
  bn_bwd_dz_kernel<T><<<ceil_div(M * cv, 256), 256, 0, cu(stream)>>>((const T*)dy, dy_ld, (const T*)y, y_ld, (const T*)z, z_ld, M, C,
                                                                     mean, rstd, relu, coef, (T*)dz, dz_ld);
  STEP_LAUNCH_CHECK("bn_bwd_dz_kernel");
  return 0;
}

// ---- the split entries: one rank's part of a reduction, and the merge of every rank's parts (synchronised BatchNorm) ----
template <typename T>
int bn_stats_local_launch(const void* z, int z_ld, long long M, int C, float* stats, int stats_ld, void* workspace, size_t ws_bytes,
                          step_stream_t stream) {
  constexpr int V = Vec16<T>::N;
  STEP_CHECK_ARG(z && stats && workspace && C > 0 && M > 0 && stats_ld >= C, "bn_stats_local: bad arguments (M=%lld C=%d stats_ld=%d)",
                 M, C, stats_ld);
  STEP_CHECK_ARG(C % V == 0 && z_ld % V == 0 && z_ld >= C, "bn_stats_local: C and z_ld must be multiples of %d, z_ld >= C (C=%d z_ld=%d)",
                 V, C, z_ld);
  STEP_CHECK_ARG(aligned16(z), "bn_stats_local: z must be 16-byte aligned");
  const size_t need = step_bn_stats_workspace_bytes(M, C);
  if (ws_bytes < need) return fail(STEP_E_WORKSPACE, "bn_stats_local: workspace %zu < %zu", ws_bytes, need);
  const int cv = C / V, cols = cv < 256 ? cv : 256, rows = 256 / cols;
  const int chunks = bn_chunks(M);
  const long long rows_per_chunk = (M + chunks - 1) / chunks;
  bn_stats_partial_kernel<T><<<dim3(chunks, ceil_div(cv, cols)), 256, 0, cu(stream)>>>((const T*)z, z_ld, M, C, cols, rows,
                                                                                        rows_per_chunk, (float*)workspace);
  STEP_LAUNCH_CHECK("bn_stats_partial_kernel");
  bn_stats_final_kernel<<<ceil_div(C, kFinalWarps), 32 * kFinalWarps, 0, cu(stream)>>>((const float*)workspace, chunks, C, C, M, nullptr,
                                                                                       nullptr, 0.0f, 0.0f, nullptr, nullptr, nullptr,
                                                                                       nullptr, nullptr, nullptr, stats, stats_ld);
  STEP_LAUNCH_CHECK("bn_stats_final_kernel");
  return 0;
}

template <typename T>
int bn_bwd_sums_launch(const void* dy, int dy_ld, const void* y, int y_ld, const void* z, int z_ld, long long M, int C, const float* mean,
                       const float* rstd, int relu, float gscale, float* sums, int sums_ld, float* dgamma, float* dbeta, void* workspace,
                       size_t ws_bytes, step_stream_t stream) {
  constexpr int V = Vec16<T>::N;
  STEP_CHECK_ARG(dy && z && mean && rstd && sums && workspace && (!relu || y) && C > 0 && M > 0 && sums_ld >= C,
                 "bn_bwd_sums: bad arguments (M=%lld C=%d sums_ld=%d)", M, C, sums_ld);
  STEP_CHECK_ARG(C % V == 0 && dy_ld % V == 0 && z_ld % V == 0 && (!relu || y_ld % V == 0) && dy_ld >= C && z_ld >= C &&
                 (!relu || y_ld >= C),
                 "bn_bwd_sums: C and the ld arguments must be multiples of %d, each ld >= C (C=%d dy_ld=%d y_ld=%d z_ld=%d)", V, C, dy_ld,
                 y_ld, z_ld);
  STEP_CHECK_ARG(aligned16(dy) && aligned16(y) && aligned16(z), "bn_bwd_sums: pointers must be 16-byte aligned");
  const size_t need = step_bn_bwd_sums_workspace_bytes(M, C);
  if (ws_bytes < need) return fail(STEP_E_WORKSPACE, "bn_bwd_sums: workspace %zu < %zu", ws_bytes, need);
  const int cv = C / V, cols = cv < 256 ? cv : 256, rows = 256 / cols;
  const int chunks = bn_chunks(M);
  const long long rows_per_chunk = (M + chunks - 1) / chunks;
  float* partial = (float*)workspace;
  bn_bwd_partial_kernel<T><<<dim3(chunks, ceil_div(cv, cols)), 256, 0, cu(stream)>>>(
      (const T*)dy, dy_ld, (const T*)y, y_ld, (const T*)z, z_ld, M, C, mean, rstd, relu, cols, rows, rows_per_chunk, partial);
  STEP_LAUNCH_CHECK("bn_bwd_partial_kernel");
  bn_bwd_reduce_kernel<<<ceil_div(C, 256), 256, 0, cu(stream)>>>(partial, chunks, C, C, M, nullptr, nullptr, gscale, dgamma, dbeta, sums,
                                                                 sums_ld, nullptr);
  STEP_LAUNCH_CHECK("bn_bwd_reduce_kernel");
  return 0;
}

template <typename T>
int bn_bwd_merge_dz_launch(const float* sums, int ranks, int sums_ld, long long M_total, const void* dy, int dy_ld, const void* y,
                           int y_ld, const void* z, int z_ld, long long M, int C, const float* mean, const float* rstd, const float* gamma,
                           int relu, void* dz, int dz_ld, void* workspace, size_t ws_bytes, step_stream_t stream) {
  constexpr int V = Vec16<T>::N;
  STEP_CHECK_ARG(sums && dy && z && dz && mean && rstd && gamma && workspace && (!relu || y) && C > 0 && M > 0 && ranks > 0 &&
                 sums_ld >= C, "bn_bwd_merge_dz: bad arguments (M=%lld C=%d ranks=%d sums_ld=%d)", M, C, ranks, sums_ld);
  STEP_CHECK_ARG(M_total > 1 && M_total >= M, "bn_bwd_merge_dz: Expected more than 1 value per channel when training (M_total=%lld, "
                 "M=%lld)", M_total, M);
  STEP_CHECK_ARG(C % V == 0 && dy_ld % V == 0 && z_ld % V == 0 && dz_ld % V == 0 && (!relu || y_ld % V == 0) && dy_ld >= C &&
                 z_ld >= C && dz_ld >= C && (!relu || y_ld >= C),
                 "bn_bwd_merge_dz: C and the ld arguments must be multiples of %d, each ld >= C (C=%d dy_ld=%d y_ld=%d z_ld=%d "
                 "dz_ld=%d)", V, C, dy_ld, y_ld, z_ld, dz_ld);
  STEP_CHECK_ARG(aligned16(dy) && aligned16(y) && aligned16(z) && aligned16(dz), "bn_bwd_merge_dz: pointers must be 16-byte aligned");
  const size_t need = step_bn_bwd_merge_dz_workspace_bytes(C);
  if (ws_bytes < need) return fail(STEP_E_WORKSPACE, "bn_bwd_merge_dz: workspace %zu < %zu", ws_bytes, need);
  float* coef = (float*)workspace;
  bn_bwd_reduce_kernel<<<ceil_div(C, 256), 256, 0, cu(stream)>>>(sums, ranks, sums_ld, C, M_total, gamma, rstd, 0.0f, nullptr, nullptr,
                                                                 nullptr, 0, coef);
  STEP_LAUNCH_CHECK("bn_bwd_reduce_kernel");
  bn_bwd_dz_kernel<T><<<ceil_div(M * (C / V), 256), 256, 0, cu(stream)>>>((const T*)dy, dy_ld, (const T*)y, y_ld, (const T*)z, z_ld, M,
                                                                          C, mean, rstd, relu, coef, (T*)dz, dz_ld);
  STEP_LAUNCH_CHECK("bn_bwd_dz_kernel");
  return 0;
}

}  // namespace

extern "C" size_t step_bn_stats_workspace_bytes(long long M, int C) {
  if (M <= 0 || C <= 0) return 0;
  return (size_t)bn_chunks(M) * 3 * C * sizeof(float);
}

extern "C" int step_bn_stats_f16(const void* z, int z_ld, long long M, int C, const float* gamma, const float* beta, float eps,
                                 float momentum, float* running_mean, float* running_var, float* mean, float* rstd, float* scale,
                                 float* shift, void* workspace, size_t ws_bytes, step_stream_t stream) {
  return bn_stats_launch<__half>(z, z_ld, M, C, gamma, beta, eps, momentum, running_mean, running_var, mean, rstd, scale, shift,
                                 workspace, ws_bytes, stream);
}

extern "C" int step_bn_stats_f32(const float* z, int z_ld, long long M, int C, const float* gamma, const float* beta, float eps,
                                 float momentum, float* running_mean, float* running_var, float* mean, float* rstd, float* scale,
                                 float* shift, void* workspace, size_t ws_bytes, step_stream_t stream) {
  return bn_stats_launch<float>(z, z_ld, M, C, gamma, beta, eps, momentum, running_mean, running_var, mean, rstd, scale, shift,
                                workspace, ws_bytes, stream);
}

extern "C" int step_bn_apply_f16(const void* z, int z_ld, long long M, int C, const float* scale, const float* shift, int relu, void* y,
                                 int y_ld, int split1, void* y1, int y1_ld, int split2, void* y2, int y2_ld, step_stream_t stream) {
  return bn_apply_launch<__half>(z, z_ld, M, C, scale, shift, relu, y, y_ld, split1, y1, y1_ld, split2, y2, y2_ld, stream);
}

extern "C" int step_bn_apply_f32(const float* z, int z_ld, long long M, int C, const float* scale, const float* shift, int relu,
                                 float* y, int y_ld, int split1, float* y1, int y1_ld, int split2, float* y2, int y2_ld,
                                 step_stream_t stream) {
  return bn_apply_launch<float>(z, z_ld, M, C, scale, shift, relu, y, y_ld, split1, y1, y1_ld, split2, y2, y2_ld, stream);
}

extern "C" size_t step_bn_bwd_workspace_bytes(long long M, int C) {
  if (M <= 0 || C <= 0) return 0;
  return ((size_t)bn_chunks(M) * 2 + 3) * C * sizeof(float);
}

extern "C" int step_bn_bwd_f16(const void* dy, int dy_ld, const void* y, int y_ld, const void* z, int z_ld, long long M, int C,
                               const float* mean, const float* rstd, const float* gamma, int relu, float gscale, void* dz, int dz_ld,
                               float* dgamma, float* dbeta, void* workspace, size_t ws_bytes, step_stream_t stream) {
  return bn_bwd_launch<__half>(dy, dy_ld, y, y_ld, z, z_ld, M, C, mean, rstd, gamma, relu, gscale, dz, dz_ld, dgamma, dbeta, workspace,
                               ws_bytes, stream);
}

extern "C" int step_bn_bwd_f32(const float* dy, int dy_ld, const float* y, int y_ld, const float* z, int z_ld, long long M, int C,
                               const float* mean, const float* rstd, const float* gamma, int relu, float gscale, float* dz, int dz_ld,
                               float* dgamma, float* dbeta, void* workspace, size_t ws_bytes, step_stream_t stream) {
  return bn_bwd_launch<float>(dy, dy_ld, y, y_ld, z, z_ld, M, C, mean, rstd, gamma, relu, gscale, dz, dz_ld, dgamma, dbeta, workspace,
                              ws_bytes, stream);
}

extern "C" int step_bn_stats_local_f16(const void* z, int z_ld, long long M, int C, float* stats, int stats_ld, void* workspace,
                                       size_t ws_bytes, step_stream_t stream) {
  return bn_stats_local_launch<__half>(z, z_ld, M, C, stats, stats_ld, workspace, ws_bytes, stream);
}

extern "C" int step_bn_stats_local_f32(const float* z, int z_ld, long long M, int C, float* stats, int stats_ld, void* workspace,
                                       size_t ws_bytes, step_stream_t stream) {
  return bn_stats_local_launch<float>(z, z_ld, M, C, stats, stats_ld, workspace, ws_bytes, stream);
}

extern "C" int step_bn_stats_merge(const float* stats, int ranks, int stats_ld, long long M, int C, const float* gamma, const float* beta,
                                   float eps, float momentum, float* running_mean, float* running_var, float* mean, float* rstd,
                                   float* scale, float* shift, step_stream_t stream) {
  STEP_CHECK_ARG(stats && gamma && beta && mean && rstd && scale && shift && C > 0 && ranks > 0 && stats_ld >= C,
                 "bn_stats_merge: bad arguments (C=%d ranks=%d stats_ld=%d)", C, ranks, stats_ld);
  STEP_CHECK_ARG(M > 1, "bn_stats_merge: Expected more than 1 value per channel when training (M=%lld)", M);
  STEP_CHECK_ARG(!running_mean == !running_var, "bn_stats_merge: give both running statistics or neither");
  STEP_CHECK_ARG(eps > 0.0f && momentum >= 0.0f && momentum <= 1.0f, "bn_stats_merge: eps %g must be > 0 and momentum %g in [0, 1]",
                 eps, momentum);
  bn_stats_final_kernel<<<ceil_div(C, kFinalWarps), 32 * kFinalWarps, 0, cu(stream)>>>(stats, ranks, stats_ld, C, M, gamma, beta, eps,
                                                                                       momentum, running_mean, running_var, mean, rstd,
                                                                                       scale, shift, nullptr, 0);
  STEP_LAUNCH_CHECK("bn_stats_final_kernel");
  return 0;
}

extern "C" size_t step_bn_bwd_sums_workspace_bytes(long long M, int C) {
  if (M <= 0 || C <= 0) return 0;
  return (size_t)bn_chunks(M) * 2 * C * sizeof(float);
}

extern "C" int step_bn_bwd_sums_f16(const void* dy, int dy_ld, const void* y, int y_ld, const void* z, int z_ld, long long M, int C,
                                    const float* mean, const float* rstd, int relu, float gscale, float* sums, int sums_ld,
                                    float* dgamma, float* dbeta, void* workspace, size_t ws_bytes, step_stream_t stream) {
  return bn_bwd_sums_launch<__half>(dy, dy_ld, y, y_ld, z, z_ld, M, C, mean, rstd, relu, gscale, sums, sums_ld, dgamma, dbeta, workspace,
                                    ws_bytes, stream);
}

extern "C" int step_bn_bwd_sums_f32(const float* dy, int dy_ld, const float* y, int y_ld, const float* z, int z_ld, long long M, int C,
                                    const float* mean, const float* rstd, int relu, float gscale, float* sums, int sums_ld,
                                    float* dgamma, float* dbeta, void* workspace, size_t ws_bytes, step_stream_t stream) {
  return bn_bwd_sums_launch<float>(dy, dy_ld, y, y_ld, z, z_ld, M, C, mean, rstd, relu, gscale, sums, sums_ld, dgamma, dbeta, workspace,
                                   ws_bytes, stream);
}

extern "C" size_t step_bn_bwd_merge_dz_workspace_bytes(int C) {
  return C > 0 ? (size_t)3 * C * sizeof(float) : 0;
}

extern "C" int step_bn_bwd_merge_dz_f16(const float* sums, int ranks, int sums_ld, long long M_total, const void* dy, int dy_ld,
                                        const void* y, int y_ld, const void* z, int z_ld, long long M, int C, const float* mean,
                                        const float* rstd, const float* gamma, int relu, void* dz, int dz_ld, void* workspace,
                                        size_t ws_bytes, step_stream_t stream) {
  return bn_bwd_merge_dz_launch<__half>(sums, ranks, sums_ld, M_total, dy, dy_ld, y, y_ld, z, z_ld, M, C, mean, rstd, gamma, relu, dz,
                                        dz_ld, workspace, ws_bytes, stream);
}

extern "C" int step_bn_bwd_merge_dz_f32(const float* sums, int ranks, int sums_ld, long long M_total, const float* dy, int dy_ld,
                                        const float* y, int y_ld, const float* z, int z_ld, long long M, int C, const float* mean,
                                        const float* rstd, const float* gamma, int relu, float* dz, int dz_ld, void* workspace,
                                        size_t ws_bytes, step_stream_t stream) {
  return bn_bwd_merge_dz_launch<float>(sums, ranks, sums_ld, M_total, dy, dy_ld, y, y_ld, z, z_ld, M, C, mean, rstd, gamma, relu, dz,
                                       dz_ld, workspace, ws_bytes, stream);
}
