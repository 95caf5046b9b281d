// gather_probe.cu -- microbenchmark behind the Take design: random 8-byte gathers per second as
// a function of table size (TLB reach / L2 residency) and of gathers in flight per lane.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o gather_probe gather_probe.cu
// Run: ./gather_probe (table-size sweep), ./gather_probe band (banded sweep of a partitioned gather, below),
// ./gather_probe requests (random requests per row in a banded gather) or ./gather_probe foldunder (folding each band
// to float32 inside the gather pass, ahead of the gathers)
#include <cstdio>
#include <cstdint>
#include <string>
#include <cuda_runtime.h>

__device__ __forceinline__ uint64_t mix(uint64_t k) {
  k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33; return k;
}

template <int U>
__global__ void gather_kernel(const uint64_t* __restrict__ vals, const int64_t* __restrict__ idx, uint64_t* __restrict__ out,
                              int64_t n, uint64_t mask, int64_t window_rows) {
  int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t base = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; base < n; base += stride * U) {
    int64_t j[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      int64_t i = base + u * stride;
      j[u] = i < n ? (idx ? idx[i] : (int64_t)(mix(i) & mask)) : 0;
      if (window_rows) j[u] = (j[u] % window_rows) + (i / window_rows) % ((mask + 1) / window_rows) * window_rows;
    }
    uint64_t v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) v[u] = vals[j[u]];
#pragma unroll
    for (int u = 0; u < U; ++u) { int64_t i = base + u * stride; if (i < n) out[i] = v[u]; }
  }
}

__global__ void fill_idx(int64_t* idx, int64_t n, uint64_t mask) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) idx[i] = mix(i * 7 + 1) & mask;
}

template <int U>
float run(const uint64_t* vals, const int64_t* idx, uint64_t* out, int64_t n, uint64_t mask, int64_t window, int blocks) {
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  gather_kernel<U><<<blocks, 256>>>(vals, idx, out, n, mask, window);
  cudaEventRecord(a);
  for (int r = 0; r < 3; ++r) gather_kernel<U><<<blocks, 256>>>(vals, idx, out, n, mask, window);
  cudaEventRecord(b); cudaEventSynchronize(b);
  float ms; cudaEventElapsedTime(&ms, a, b); return ms / 3;
}

// ---- pass-B model of a partitioned gather --------------------------------------------------------------------------
// Rows arrive grouped by band (band b = rows [b*n/nb, (b+1)*n/nb)), each row carrying a uint32 offset inside its band,
// as the partition pass of a partitioned Take would leave them.  Tiles are claimed through an atomic ticket so the
// sweep walks the bands in order.  pf = 0: no prefetch; 1: every tile bulk-prefetches its share of the NEXT band into
// L2 (cp.async.bulk.prefetch.L2), so band b+1 is read from DRAM sequentially while band b is gathered; 2: as 1 with
// the prefetch evict_last and the gathers evict_first (a gathered band leaves L2 first).  Writes 4 B per row (the cast
// result), like the pass it models.
constexpr int kBandThreads = 256, kBandItems = 8, kBandTile = kBandThreads * kBandItems;

__global__ void fill_band_off(uint32_t* off, int64_t n, int64_t nb, int64_t band_rows, int64_t table_rows) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i * nb / n;
    const int64_t len = table_rows - b * band_rows < band_rows ? table_rows - b * band_rows : band_rows;
    off[i] = (uint32_t)(mix(i * 7 + 1) % (uint64_t)len);
  }
}

template <int PF>
__global__ void __launch_bounds__(kBandThreads) band_gather_kernel(const double* __restrict__ vals, const uint32_t* __restrict__ off,
                                                                   float* __restrict__ out, int64_t n, int64_t nb, int64_t band_rows,
                                                                   int64_t table_rows, unsigned* ticket) {
  __shared__ unsigned s_tile;
  uint64_t pol_first, pol_last;
  asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol_first));
  asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol_last));
  const int64_t n_tiles = (n + kBandTile - 1) / kBandTile;
  for (;;) {
    __syncthreads();
    if (threadIdx.x == 0) s_tile = atomicAdd(ticket, 1u);
    __syncthreads();
    const int64_t tile = s_tile;
    if (tile >= n_tiles) return;
    const int64_t r0 = tile * kBandTile;
    if (PF && threadIdx.x == 0) {
      // rows map onto the table in order, table_rows / n rows of table per row: prefetch the slice one band ahead
      const int64_t ahead = n / nb;
      const int64_t lo = (r0 + ahead) * table_rows / n, hi = (r0 + ahead + kBandTile) * table_rows / n;
      const int64_t lo16 = lo & ~int64_t(1), hi16 = (hi < table_rows ? hi : table_rows) & ~int64_t(1);
      if (hi16 > lo16) {
        const double* p = vals + lo16;
        const unsigned bytes = (unsigned)((hi16 - lo16) * 8);
        if (PF == 1) asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p), "r"(bytes) : "memory");
        else asm volatile("cp.async.bulk.prefetch.L2.global.L2::cache_hint [%0], %1, %2;" ::"l"(p), "r"(bytes), "l"(pol_last) : "memory");
      }
    }
    uint32_t o[kBandItems];
#pragma unroll
    for (int k = 0; k < kBandItems; ++k) {
      const int64_t i = r0 + k * kBandThreads + threadIdx.x;
      o[k] = i < n ? __ldcs(off + i) : 0;
    }
    double v[kBandItems];
#pragma unroll
    for (int k = 0; k < kBandItems; ++k) {
      const int64_t i = r0 + k * kBandThreads + threadIdx.x;
      const int64_t b = (i < n ? i : n - 1) * nb / n;
      const double* p = vals + b * band_rows + o[k];
      if (PF == 2) asm volatile("ld.global.nc.L2::cache_hint.f64 %0, [%1], %2;" : "=d"(v[k]) : "l"(p), "l"(pol_first));
      else v[k] = __ldg(p);
    }
#pragma unroll
    for (int k = 0; k < kBandItems; ++k) {
      const int64_t i = r0 + k * kBandThreads + threadIdx.x;
      if (i < n) __stcs(out + i, (float)v[k]);
    }
  }
}

static void run_band_probe() {
  const int64_t n = 1ll << 30, table_rows = 1ll << 30;  // 1G gathers into an 8 GB float64 table (the bench shape)
  double* vals; uint32_t* off; float* out; unsigned* ticket;
  cudaMalloc(&vals, table_rows * 8); cudaMalloc(&off, n * 4); cudaMalloc(&out, n * 4); cudaMalloc(&ticket, 4);
  cudaMemset(vals, 1, table_rows * 8);
  int dev = 0, sms = 0, per_sm = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, band_gather_kernel<0>, kBandThreads, 0);
  const int grid = sms * per_sm;
  printf("band_MB,prefetch,ms,Ggathers_per_s\n");
  for (int64_t band_mb : {8, 16, 24, 32, 8192}) {  // 8192: one band = fully random gathers over the whole table
    const int64_t band_rows = (band_mb << 20) / 8;
    const int64_t nb = (table_rows + band_rows - 1) / band_rows;
    fill_band_off<<<sms * 8, 256>>>(off, n, nb, band_rows, table_rows);
    for (int pf = 0; pf < (nb > 1 ? 3 : 1); ++pf) {
      auto launch = [&] {
        cudaMemsetAsync(ticket, 0, 4);
        if (pf == 0) band_gather_kernel<0><<<grid, kBandThreads>>>(vals, off, out, n, nb, band_rows, table_rows, ticket);
        else if (pf == 1) band_gather_kernel<1><<<grid, kBandThreads>>>(vals, off, out, n, nb, band_rows, table_rows, ticket);
        else band_gather_kernel<2><<<grid, kBandThreads>>>(vals, off, out, n, nb, band_rows, table_rows, ticket);
      };
      launch();
      cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
      float best = 1e30f;
      for (int r = 0; r < 5; ++r) {
        cudaEventRecord(a); launch(); cudaEventRecord(b); cudaEventSynchronize(b);
        float ms; cudaEventElapsedTime(&ms, a, b); best = ms < best ? ms : best;
      }
      printf("%lld,%d,%.3f,%.1f\n", (long long)band_mb, pf, best, n / best / 1e6);
    }
  }
  cudaFree(vals); cudaFree(off); cudaFree(out); cudaFree(ticket);
}

// ---- random requests per row in a banded gather ----------------------------------------------------------------------
// The same banded sweep (no prefetch), 4M-row bands of a 1G-row table, in four request patterns:
//   0  one 8 B gather per row from a 32 MB float64 band
//   1  one 4 B gather per row from a 16 MB float32 band
//   2  as 0 plus a 1-byte probe into the band's 512 KB slice of a validity bitmap: the partitioned Take's pass B today
//   3  as 1 plus, for 10 % of the rows, a 4 B read from the band's 1.6 MB slice of a side table: the folded pass B
template <int MODE>
__global__ void __launch_bounds__(kBandThreads) band_requests_kernel(const void* __restrict__ table, const uint8_t* __restrict__ bits,
                                                                     const float* __restrict__ side, const uint32_t* __restrict__ off,
                                                                     float* __restrict__ out, int64_t n, int64_t nb, int64_t band_rows,
                                                                     int64_t side_rows, unsigned* ticket) {
  __shared__ unsigned s_tile;
  const int64_t n_tiles = (n + kBandTile - 1) / kBandTile;
  for (;;) {
    __syncthreads();
    if (threadIdx.x == 0) s_tile = atomicAdd(ticket, 1u);
    __syncthreads();
    const int64_t tile = s_tile;
    if (tile >= n_tiles) return;
    const int64_t r0 = tile * kBandTile;
    uint32_t o[kBandItems];
    int64_t b[kBandItems];
#pragma unroll
    for (int k = 0; k < kBandItems; ++k) {
      const int64_t i = r0 + k * kBandThreads + threadIdx.x;
      o[k] = i < n ? __ldcs(off + i) : 0;
      b[k] = (i < n ? i : n - 1) * nb / n;
    }
    float v[kBandItems];
    uint32_t x[kBandItems];
#pragma unroll
    for (int k = 0; k < kBandItems; ++k) {
      const int64_t j = b[k] * band_rows + o[k];
      if (MODE == 0 || MODE == 2) v[k] = (float)__ldg(static_cast<const double*>(table) + j);
      else v[k] = __ldg(static_cast<const float*>(table) + j);
      if (MODE == 2) x[k] = __ldg(bits + (j >> 3));
    }
#pragma unroll
    for (int k = 0; k < kBandItems; ++k) {
      if (MODE == 2) v[k] += (float)((x[k] >> (o[k] & 7)) & 1u);
      if (MODE == 3 && o[k] % 10 == 0) v[k] += __ldg(side + b[k] * side_rows + (o[k] / 10) % side_rows);
    }
#pragma unroll
    for (int k = 0; k < kBandItems; ++k) {
      const int64_t i = r0 + k * kBandThreads + threadIdx.x;
      if (i < n) __stcs(out + i, v[k]);
    }
  }
}

static void run_requests_probe() {
  const int64_t n = 1ll << 30, table_rows = 1ll << 30, band_rows = 1ll << 22, side_rows = band_rows / 10;
  const int64_t nb = table_rows / band_rows;
  void* table; uint8_t* bits; float* side; uint32_t* off; float* out; unsigned* ticket;
  cudaMalloc(&table, table_rows * 8); cudaMalloc(&bits, table_rows / 8); cudaMalloc(&side, nb * side_rows * 4);
  cudaMalloc(&off, n * 4); cudaMalloc(&out, n * 4); cudaMalloc(&ticket, 4);
  cudaMemset(table, 1, table_rows * 8); cudaMemset(bits, 0xff, table_rows / 8); cudaMemset(side, 0, nb * side_rows * 4);
  int dev = 0, sms = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  fill_band_off<<<sms * 8, 256>>>(off, n, nb, band_rows, table_rows);
  const char* names[4] = {"8B gather, 32 MB band", "4B gather, 16 MB band", "8B gather + bitmap byte", "4B gather + 10% side"};
  printf("mode,pattern,ms,Grows_per_s,Grequests_per_s\n");
  for (int mode = 0; mode < 4; ++mode) {
    int per_sm = 0;
    if (mode == 0) cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, band_requests_kernel<0>, kBandThreads, 0);
    if (mode == 1) cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, band_requests_kernel<1>, kBandThreads, 0);
    if (mode == 2) cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, band_requests_kernel<2>, kBandThreads, 0);
    if (mode == 3) cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, band_requests_kernel<3>, kBandThreads, 0);
    const int grid = sms * per_sm;
    auto launch = [&] {
      cudaMemsetAsync(ticket, 0, 4);
      if (mode == 0) band_requests_kernel<0><<<grid, kBandThreads>>>(table, bits, side, off, out, n, nb, band_rows, side_rows, ticket);
      if (mode == 1) band_requests_kernel<1><<<grid, kBandThreads>>>(table, bits, side, off, out, n, nb, band_rows, side_rows, ticket);
      if (mode == 2) band_requests_kernel<2><<<grid, kBandThreads>>>(table, bits, side, off, out, n, nb, band_rows, side_rows, ticket);
      if (mode == 3) band_requests_kernel<3><<<grid, kBandThreads>>>(table, bits, side, off, out, n, nb, band_rows, side_rows, ticket);
    };
    launch();
    cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
    float best = 1e30f;
    for (int r = 0; r < 5; ++r) {
      cudaEventRecord(a); launch(); cudaEventRecord(b); cudaEventSynchronize(b);
      float ms; cudaEventElapsedTime(&ms, a, b); best = ms < best ? ms : best;
    }
    const double reqs = mode == 2 ? 2.0 : mode == 3 ? 1.1 : 1.0;
    printf("%d,%s,%.3f,%.1f,%.1f\n", mode, names[mode], best, n / best / 1e6, reqs * n / best / 1e6);
  }
  cudaFree(table); cudaFree(bits); cudaFree(side); cudaFree(off); cudaFree(out); cudaFree(ticket);
}

// ---- fold under the gather -------------------------------------------------------------------------------------------
// Models folding each band of a float64 table to float32 inside the banded gather pass, L bands ahead of the gather
// front, against the two passes run one after the other.  1G rows grouped by band, 1G values, 2^22-row bands, 4096-row
// items, one item per CTA claimed in order through a ticket.  A fold item streams 4096 values in and stores their
// float32 casts with plain stores (the band should stay in L2); a gather item reads 4096 band offsets, gathers from
// the folded band through L2 (ld.global.cg: another CTA of the same launch wrote it) and streams 4 B per row out.  A
// fold CTA counts itself into its band's counter after a fence; a gather CTA waits for its band's 1024.  Every fold
// item a gather item waits on has a smaller ticket, and a ticket is only ever held by a running CTA, so the wait ends
// whatever the residency; it also gives up after kWaitBudgetNs and sets a flag, which fails the run.
// MIX = 0: each step is band g+L's fold items, then band g's gather items; 1: the two alternate within the step.
constexpr int kFuItem = 4096, kFuItems = kFuItem / kBandThreads, kFuBandLog2 = 22, kFuBands = 256;
constexpr int kFuPerBand = (1 << kFuBandLog2) / kFuItem;  // items of either kind per band
constexpr unsigned long long kWaitBudgetNs = 2000000000ull;

__device__ __forceinline__ void fu_fold_item(const double* __restrict__ vals, uint32_t* __restrict__ folded, uint32_t item) {
  const int64_t base = (int64_t)item * kFuItem;
  double v[kFuItems];
#pragma unroll
  for (int k = 0; k < kFuItems; ++k) v[k] = __ldcs(vals + base + k * kBandThreads + threadIdx.x);
#pragma unroll
  for (int k = 0; k < kFuItems; ++k) folded[base + k * kBandThreads + threadIdx.x] = __float_as_uint((float)v[k]);
}

template <bool CG>
__device__ __forceinline__ void fu_gather_item(const uint32_t* __restrict__ folded, const uint32_t* __restrict__ off,
                                               float* __restrict__ out, uint32_t item, const unsigned* done, unsigned* stalled) {
  const int64_t p0 = (int64_t)item * kFuItem;
  const uint32_t band = item / kFuPerBand;
  uint32_t o[kFuItems];
#pragma unroll
  for (int k = 0; k < kFuItems; ++k) o[k] = __ldcs(off + p0 + k * kBandThreads + threadIdx.x);
  if (done) {
    if (threadIdx.x == 0) {
      unsigned long long t0 = 0, now;
      for (;;) {
        unsigned seen;
        asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(seen) : "l"(done + band) : "memory");
        if (seen >= (unsigned)kFuPerBand) break;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
        if (!t0) t0 = now;
        if (now - t0 > kWaitBudgetNs || *(volatile unsigned*)stalled) { *stalled = 1u; break; }
        __nanosleep(200);
      }
    }
    __syncthreads();
  }
  const uint32_t* b = folded + ((int64_t)band << kFuBandLog2);
  uint32_t x[kFuItems];
#pragma unroll
  for (int k = 0; k < kFuItems; ++k) {
    if (CG) asm volatile("ld.global.cg.u32 %0, [%1];" : "=r"(x[k]) : "l"(b + o[k]));
    else asm volatile("ld.global.u32 %0, [%1];" : "=r"(x[k]) : "l"(b + o[k]));
  }
#pragma unroll
  for (int k = 0; k < kFuItems; ++k) __stcs(out + p0 + k * kBandThreads + threadIdx.x, __uint_as_float(x[k]));
}

__global__ void __launch_bounds__(kBandThreads) fu_fold_all_kernel(const double* __restrict__ vals, uint32_t* __restrict__ folded) {
  fu_fold_item(vals, folded, blockIdx.x);
}

__global__ void __launch_bounds__(kBandThreads) fu_gather_all_kernel(const uint32_t* __restrict__ folded, const uint32_t* __restrict__ off,
                                                                     float* __restrict__ out, unsigned* ticket) {
  __shared__ unsigned s_item;
  if (threadIdx.x == 0) s_item = atomicAdd(ticket, 1u);
  __syncthreads();
  fu_gather_item<false>(folded, off, out, s_item, nullptr, nullptr);
}

// ctl: [0] the ticket, [1 .. 256] the bands' fold counters, [257] the stalled flag
template <int L, bool MIX>
__global__ void __launch_bounds__(kBandThreads) fu_fused_kernel(const double* __restrict__ vals, uint32_t* folded,
                                                                const uint32_t* __restrict__ off, float* __restrict__ out,
                                                                unsigned* ctl) {
  __shared__ unsigned s_item;
  if (threadIdx.x == 0) s_item = atomicAdd(ctl, 1u);
  __syncthreads();
  const uint32_t t = s_item;
  bool is_fold;
  uint32_t item;
  constexpr uint32_t kHead = L * kFuPerBand, kSteady = (kFuBands - L) * 2 * kFuPerBand;
  if (t < kHead) {
    is_fold = true, item = t;
  } else if (t - kHead < kSteady) {
    const uint32_t u = t - kHead, g = u / (2 * kFuPerBand), r = u % (2 * kFuPerBand);
    is_fold = MIX ? (r & 1u) == 0 : r < (uint32_t)kFuPerBand;
    const uint32_t i = MIX ? r >> 1 : r % kFuPerBand;
    item = (is_fold ? g + L : g) * kFuPerBand + i;
  } else {
    is_fold = false, item = (kFuBands - L) * kFuPerBand + (t - kHead - kSteady);
  }
  if (is_fold) {
    fu_fold_item(vals, folded, item);
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) atomicAdd(ctl + 1 + item / kFuPerBand, 1u);
  } else {
    fu_gather_item<true>(folded, off, out, item, ctl + 1, ctl + 1 + kFuBands);
  }
}

static int run_fold_under_probe() {
  const int64_t n = 1ll << 30, table_rows = 1ll << 30, band_rows = 1ll << kFuBandLog2;
  const uint32_t items = (uint32_t)(n / kFuItem);
  double* vals; uint32_t* folded; uint32_t* off; float* out; unsigned* ctl;
  cudaMalloc(&vals, table_rows * 8); cudaMalloc(&folded, table_rows * 4); cudaMalloc(&off, n * 4); cudaMalloc(&out, n * 4);
  cudaMalloc(&ctl, (kFuBands + 2) * 4);
  cudaMemset(vals, 1, table_rows * 8);
  int dev = 0, sms = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  fill_band_off<<<sms * 8, 256>>>(off, n, kFuBands, band_rows, table_rows);
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  auto best_of = [&](auto launch) {
    launch();
    float best = 1e30f;
    for (int r = 0; r < 5; ++r) {
      cudaEventRecord(a); launch(); cudaEventRecord(b); cudaEventSynchronize(b);
      float ms; cudaEventElapsedTime(&ms, a, b); best = ms < best ? ms : best;
    }
    return best;
  };
  printf("kernel,lead_bands,interleaved,ms\n");
  const float t_fold = best_of([&] { fu_fold_all_kernel<<<items, kBandThreads>>>(vals, folded); });
  const float t_gather = best_of([&] {
    cudaMemsetAsync(ctl, 0, 4);
    fu_gather_all_kernel<<<items, kBandThreads>>>(folded, off, out, ctl);
  });
  const float t_both = best_of([&] {
    cudaMemsetAsync(ctl, 0, 4);
    fu_fold_all_kernel<<<items, kBandThreads>>>(vals, folded);
    fu_gather_all_kernel<<<items, kBandThreads>>>(folded, off, out, ctl);
  });
  printf("fold,-,-,%.3f\ngather,-,-,%.3f\nfold then gather,-,-,%.3f\n", t_fold, t_gather, t_both);
  int lead = 0, mix = 0;
  auto fused = [&] {
    cudaMemsetAsync(ctl, 0, (kFuBands + 2) * 4);
    if (lead == 1 && !mix) fu_fused_kernel<1, false><<<2 * items, kBandThreads>>>(vals, folded, off, out, ctl);
    if (lead == 2 && !mix) fu_fused_kernel<2, false><<<2 * items, kBandThreads>>>(vals, folded, off, out, ctl);
    if (lead == 4 && !mix) fu_fused_kernel<4, false><<<2 * items, kBandThreads>>>(vals, folded, off, out, ctl);
    if (lead == 1 && mix) fu_fused_kernel<1, true><<<2 * items, kBandThreads>>>(vals, folded, off, out, ctl);
    if (lead == 2 && mix) fu_fused_kernel<2, true><<<2 * items, kBandThreads>>>(vals, folded, off, out, ctl);
    if (lead == 4 && mix) fu_fused_kernel<4, true><<<2 * items, kBandThreads>>>(vals, folded, off, out, ctl);
  };
  unsigned stalled = 0;
  for (mix = 0; mix < 2 && !stalled; ++mix)
    for (lead = 1; lead <= 4 && !stalled; lead *= 2) {
      const float t = best_of(fused);
      cudaMemcpy(&stalled, ctl + 1 + kFuBands, 4, cudaMemcpyDeviceToHost);
      printf("fused,%d,%d,%.3f%s\n", lead, mix, t, stalled ? " STALLED" : "");
    }
  cudaFree(vals); cudaFree(folded); cudaFree(off); cudaFree(out); cudaFree(ctl);
  return stalled ? 1 : 0;
}

int main(int argc, char** argv) {
  if (argc > 1 && std::string(argv[1]) == "foldunder") {
    const int stalled = run_fold_under_probe();
    cudaError_t e = cudaDeviceSynchronize();
    printf("# %s\n", cudaGetErrorString(e));
    return e == cudaSuccess && !stalled ? 0 : 1;
  }
  if (argc > 1 && std::string(argv[1]) == "requests") {
    run_requests_probe();
    cudaError_t e = cudaDeviceSynchronize();
    printf("# %s\n", cudaGetErrorString(e));
    return e == cudaSuccess ? 0 : 1;
  }
  if (argc > 1 && std::string(argv[1]) == "band") {
    run_band_probe();
    cudaError_t e = cudaDeviceSynchronize();
    printf("# %s\n", cudaGetErrorString(e));
    return e == cudaSuccess ? 0 : 1;
  }
  const int64_t n = 1ll << 28;  // 268M gathers per launch
  uint64_t *vals, *out; int64_t* idx;
  cudaMalloc(&vals, 8ull << 30); cudaMalloc(&out, n * 8); cudaMalloc(&idx, n * 8);
  cudaMemset(vals, 1, 8ull << 30);
  printf("table_MB,U,idx_in_mem,window_MB,ms,Ggathers_per_s\n");
  for (int shift = 23; shift <= 30; ++shift) {  // table rows 2^shift * 8 B = 64 MB .. 8 GB
    uint64_t mask = (1ull << shift) - 1;
    fill_idx<<<132 * 8, 256>>>(idx, n, mask);
    for (int mem = 0; mem < 2; ++mem) {
      float t4 = run<4>(vals, mem ? idx : nullptr, out, n, mask, 0, 132 * 16);
      float t8 = run<8>(vals, mem ? idx : nullptr, out, n, mask, 0, 132 * 16);
      float t16 = run<16>(vals, mem ? idx : nullptr, out, n, mask, 0, 132 * 16);
      printf("%llu,4,%d,0,%.3f,%.1f\n", (unsigned long long)((mask + 1) * 8 >> 20), mem, t4, n / t4 / 1e6);
      printf("%llu,8,%d,0,%.3f,%.1f\n", (unsigned long long)((mask + 1) * 8 >> 20), mem, t8, n / t8 / 1e6);
      printf("%llu,16,%d,0,%.3f,%.1f\n", (unsigned long long)((mask + 1) * 8 >> 20), mem, t16, n / t16 / 1e6);
    }
  }
  // L2 fetch granularity hint (cudaLimitMaxL2FetchGranularity: 32 / 64 / 128 bytes), 8 GB table
  for (size_t gran : {32, 64, 128}) {
    cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, gran);
    size_t got = 0; cudaDeviceGetLimit(&got, cudaLimitMaxL2FetchGranularity);
    uint64_t m = (1ull << 30) - 1;
    float t = run<8>(vals, nullptr, out, n, m, 0, 132 * 16);
    printf("# l2_fetch_granularity req=%zu got=%zu : %.3f ms, %.1f Ggathers/s\n", gran, got, t, n / t / 1e6);
  }
  // 8 GB table, but consecutive groups of gathers confined to a window (what a partition pass would give)
  uint64_t mask = (1ull << 30) - 1;
  for (int wshift = 22; wshift <= 28; wshift += 2) {
    int64_t window = 1ll << wshift;
    float t = run<8>(vals, nullptr, out, n, mask, window, 132 * 16);
    printf("8192,8,0,%lld,%.3f,%.1f\n", (long long)(window * 8 >> 20), t, n / t / 1e6);
  }
  cudaError_t e = cudaDeviceSynchronize();
  printf("# %s\n", cudaGetErrorString(e));
  return 0;
}
