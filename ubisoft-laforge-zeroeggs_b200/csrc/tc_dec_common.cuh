// Helpers shared by the tensor-core decoder kernels (forward and backward recurrences).
#pragma once
#include "decoder_common.cuh"
#include "tc_common.cuh"

namespace zeggs {

// byte offset of element (row, k) inside an image whose k-block tiles have `rows` rows
__host__ __device__ inline size_t img_off(int rows, int row, int k) {
  const int kb = k >> 6, c = (k & 63) >> 3, e = k & 7;
  return (size_t)kb * rows * 128 + (size_t)row * 128 + (size_t)((c ^ (row & 7)) << 4) + (size_t)e * 2;
}


__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n"
               ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// ---- thread-block clusters: cluster barrier, distributed shared memory (DSMEM), mbarrier signals across the cluster
// every thread of every CTA of the cluster; not .aligned, so the threads of a warp may arrive from different branches
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release;\n" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire;\n" ::: "memory");
}
// shared::cluster address of the same shared-memory object in CTA `rank` of the cluster, and a load through such an address
// (volatile: it stays after the mbarrier wait that publishes the data)
__device__ __forceinline__ uint32_t cluster_map(const void* p, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;\n" : "=r"(r) : "r"(smem_u32(p)), "r"(rank));
  return r;
}
__device__ __forceinline__ float ld_cluster_f32(uint32_t addr) {
  float v;
  asm volatile("ld.shared::cluster.f32 %0, [%1];\n" : "=f"(v) : "r"(addr));
  return v;
}
// arrive on the mbarrier at `bar`'s offset in CTA `rank`; release at cluster scope: this thread's earlier shared-memory writes,
// and those ordered before them by a CTA barrier, are visible to a thread that then acquires the phase with mbar_wait_cluster
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t rank) {
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];\n" ::"r"(cluster_map(bar, rank)) : "memory");
}
// mbar_wait with acquire at cluster scope (the phase includes arrivals from another CTA of the cluster)
__device__ __forceinline__ void mbar_wait_cluster(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  uint32_t done = 0;
#pragma unroll 1
  for (uint32_t it = 0; it < 20000000u; ++it) {
    asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}\n"
                 : "=r"(done) : "r"(addr), "r"(parity) : "memory");
    if (done) return;
  }
  __trap();
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async;\n" ::: "memory"); }

// Stages rows [0, nrows) of a warpgroup's m64nN accumulator fragment (Wgmma<N>) as out[col * ld + row0 + row].  With ld % 32 == 4
// the stores of a warp hit 32 distinct banks, and a warp that later reads one column for 32 consecutive rows does too.
template <int N>
__device__ __forceinline__ void stage_acc(const float (&d)[N / 2], float* out, int ld, int row0, int nrows) {
  const int wq = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const int r = 16 * wq + (lane >> 2), c = 2 * (lane & 3);
#pragma unroll
  for (int i = 0; i < N / 8; ++i) {
    if (r < nrows) { out[(size_t)(8 * i + c) * ld + row0 + r] = d[4 * i]; out[(size_t)(8 * i + c + 1) * ld + row0 + r] = d[4 * i + 1]; }
    if (r + 8 < nrows) { out[(size_t)(8 * i + c) * ld + row0 + r + 8] = d[4 * i + 2]; out[(size_t)(8 * i + c + 1) * ld + row0 + r + 8] = d[4 * i + 3]; }
  }
}
// NC consecutive columns of one row of a staged accumulator
template <int NC>
__device__ __forceinline__ void acc_ld(const float* p, int ld, float (&v)[NC]) {
#pragma unroll
  for (int i = 0; i < NC; ++i) v[i] = p[(size_t)i * ld];
}

// bf16-engine gate math: exp via the SFU (relative error ~1e-6, far below the bf16 operand rounding)
__device__ __forceinline__ float fast_sigmoid(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }
__device__ __forceinline__ float fast_tanh(float x) { return 1.0f - __fdividef(2.0f, 1.0f + __expf(2.0f * x)); }

// grid barrier split in two halves: the epilogue warp arrives, the activation loader waits
__device__ __forceinline__ void grid_arrive(unsigned* counter) {
  __syncwarp();   // the lanes' stores happen-before lane 0's release (cumulative at gpu scope)
  if ((threadIdx.x & 31) == 0) asm volatile("red.release.gpu.global.add.u32 [%0], 1;\n" ::"l"(counter) : "memory");
}
__device__ __forceinline__ void grid_wait(const unsigned* counter, unsigned target) {
  long long t0 = clock64();
  while (ld_acquire_u32(counter) < target) {
    if (clock64() - t0 > 4000000000LL) __trap();
  }
}

// write U consecutive bf16 values (units j0..j0+U-1 of sample row b) into an activation image
template <int U>
__device__ __forceinline__ void store_img_units(uint8_t* img, int b, int j0, const float (&h)[U]) {
  __nv_bfloat16 t[U];
#pragma unroll
  for (int i = 0; i < U; ++i) t[i] = __float2bfloat16_rn(h[i]);
  uint8_t* p = img + img_off(32, b, j0);
  if (U == 8) *reinterpret_cast<uint4*>(p) = *reinterpret_cast<const uint4*>(t);
  else *reinterpret_cast<uint2*>(p) = *reinterpret_cast<const uint2*>(t);
}


}  // namespace zeggs
