// seed.cu — pcl_seed_rng: each selected env's generator slots as a fresh seed leaves them
// (pcl.h PCL_SEED_*, MtSeed in pcl_mt.cuh).
//
// One thread per (env, slot): the seeding recurrences are serial within a slot.  A warp's 32
// slots are 32 consecutive 625-word rows of d_rng, so a thread's own words lie 2.5 KB from
// its neighbours'.  Rather than store them that way (every warp store touching 32 lines),
// each thread puts 32 words at a time into its row of a shared-memory tile and the warp
// stores the tile one d_rng row at a time, 32 consecutive words per store.
#include "pcl_device.cuh"
#include "pcl_kernels.cuh"
#include "pcl_mt.cuh"

namespace pcl {

namespace {

constexpr int kSeedWarps = 4;

__global__ void __launch_bounds__(kSeedWarps * 32) seed_rng_kernel(const SeedParams p) {
  __shared__ uint32_t tiles[kSeedWarps][32][33];   // [lane][word]; 33 keeps both sides conflict-free
  uint32_t (*tile)[33] = tiles[threadIdx.x >> 5];
  const int lane = threadIdx.x & 31;
  const int64_t pair = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;   // env * slots + slot
  const int env = (int)(pair / p.slots), slot = (int)(pair % p.slots);
  const bool mine = pair < (int64_t)p.B * p.slots && (!p.env_mask || p.env_mask[env]);
  const unsigned selected = __ballot_sync(0xffffffffu, mine);
  if (!selected) return;
  uint32_t* rows = p.rng + (pair - lane) * PCL_MT_WORDS;                 // the warp's first row
  MtSeed seed;
  seed.start(mine ? p.seeds[env] : 0u, (p.python_slots >> slot) & 1u);
  for (int base = 0; base < 624; base += 32) {
#pragma unroll 4
    for (int k = 0; k < 32; ++k) {
      const int i = base + k;
      if (i >= 2 && i < 624) tile[lane][k] = seed.word(i);
    }
    __syncwarp();
    const int i = base + lane;
    if (i >= 2 && i < 624)
      for (int r = 0; r < 32; ++r)
        if (selected >> r & 1u) rows[r * PCL_MT_WORDS + i] = tile[r][lane];
    __syncwarp();
  }
  if (mine) {
    uint32_t* mt = p.rng + pair * PCL_MT_WORDS;
    uint32_t w0, w1;
    seed.head(&w0, &w1);
    mt[0] = w0;
    mt[1] = w1;
    mt[624] = 624;
  }
}

}  // namespace

cudaError_t launch_seed_rng(const SeedParams& p, cudaStream_t s) {
  const int64_t threads = (int64_t)p.B * p.slots;
  const int block = kSeedWarps * 32;
  seed_rng_kernel<<<(unsigned)((threads + block - 1) / block), block, 0, s>>>(p);
  return cudaGetLastError();
}

}  // namespace pcl
