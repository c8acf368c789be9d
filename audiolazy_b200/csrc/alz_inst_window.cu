// Window kernels (alz_window.cuh): one section per channel, any order / sparsity.
#include "alz_lane_tma.cuh"
#include "alz_plan.h"
#include "alz_window.cuh"

static const int kWinSmall = 64, kWinLarge = 3584;   // coefficient capacity (doubles): 2 / 112 channels
static const int kWinWarpsPerSm = 12;                // ~160 registers per thread (two 16-slot windows + a block in flight)

template <int MX, int MY, int NCOEF>
__global__ void __launch_bounds__(32, kWinWarpsPerSm)
alz_window_kernel(const __grid_constant__ AlzTileArgs a, const __grid_constant__ AlzWindowArgs<NCOEF> ca) {
  extern __shared__ __align__(16) float alz_smem[];
  alz_run_warp<AlzWindowCore<MX, MY, NCOEF>>(a, ca, alz_smem);
}

template <int MX, int MY, int NCOEF>
__global__ void __launch_bounds__(32, kWinWarpsPerSm)
alz_window_tma_kernel(const __grid_constant__ AlzTileArgs a, const __grid_constant__ AlzWindowArgs<NCOEF> ca,
                      const __grid_constant__ CUtensorMap tmx, const __grid_constant__ CUtensorMap tmy) {
  extern __shared__ __align__(1024) unsigned char alz_smem_tma[];
  alz_run_warp_tma<AlzWindowCore<MX, MY, NCOEF>>(a, ca, &tmx, &tmy, alz_smem_tma);
}

template <int MX, int MY, int NCOEF>
static int launch_window_t(const alz_plan* p, AlzTileArgs ta, cudaStream_t st) {
  const long long groups = (ta.S + 31) / 32;
  CUtensorMap tmx, tmy;
  if (alzi_make_tensor_maps(ta, &tmx, &tmy)) {
    const long long warps = (long long)p->C * groups;
    ta.paired = warps >= (long long)p->sm_count * kWinWarpsPerSm ? 2 : 1;
    ta.groups = (int)groups;
    if (alzi_env_int("ALZ_LOG_LAUNCH", 0))
      fprintf(stderr, "alz window launch: %lld warps, paired %d\n", warps, ta.paired);
    void* args[4] = {(void*)&ta, p->win_block, (void*)&tmx, (void*)&tmy};
    ALZ_CUDA(cudaLaunchKernel((const void*)alz_window_tma_kernel<MX, MY, NCOEF>, dim3((unsigned)p->C, (unsigned)groups), dim3(32), args,
                              ALZ_TMA_SMEM_FOR(ta.paired), st));
  } else {
    void* args[2] = {(void*)&ta, p->win_block};
    ALZ_CUDA(cudaLaunchKernel((const void*)alz_window_kernel<MX, MY, NCOEF>, dim3((unsigned)p->C, (unsigned)groups), dim3(32), args,
                              ALZ_WARP_SMEM, st));
  }
  ALZ_CUDA(cudaGetLastError());
  alzi_launches.fetch_add(1, std::memory_order_relaxed);
  return ALZI_OK;
}

template <int MX, int MY>
static int launch_window_n(const alz_plan* p, const AlzTileArgs& ta, cudaStream_t st) {
  return p->coef_small ? launch_window_t<MX, MY, kWinSmall>(p, ta, st) : launch_window_t<MX, MY, kWinLarge>(p, ta, st);
}

template <int MX>
static int launch_window_x(const alz_plan* p, const AlzTileArgs& ta, cudaStream_t st) {
  switch (p->win_my) {
    case 0: return launch_window_n<MX, 0>(p, ta, st);
    case 4: return launch_window_n<MX, 4>(p, ta, st);
    default: return launch_window_n<MX, 16>(p, ta, st);
  }
}

int alzi_launch_window(const alz_plan* p, const AlzTileArgs& ta, cudaStream_t st) {
  switch (p->win_mx) {
    case 0: return launch_window_x<0>(p, ta, st);
    case 4: return launch_window_x<4>(p, ta, st);
    default: return launch_window_x<16>(p, ta, st);
  }
}

size_t alzi_window_block_bytes(bool small) { return small ? sizeof(AlzWindowArgs<kWinSmall>) : sizeof(AlzWindowArgs<kWinLarge>); }

// Fill the (host) parameter block of a window plan; `far_delay` / `far_coef` are DEVICE pointers.
void alzi_window_block_fill(void* blk, bool small, int n_far_x, int n_far_y, int xbase, int xmask, int ybase, int ymask, int xwin,
                            int ywin, int C, const int* far_delay, const double* far_coef, const double* coef) {
  auto fill = [&](auto* a) {
    a->n_far_x = n_far_x; a->n_far_y = n_far_y; a->xbase = xbase; a->xmask = xmask; a->ybase = ybase; a->ymask = ymask;
    a->xwin = xwin; a->ywin = ywin; a->C = C; a->pad_ = 0; a->far_delay = far_delay; a->far_coef = far_coef;
    memcpy(a->coef, coef, (size_t)C * ALZ_WIN_REC * sizeof(double));
  };
  if (small) fill(reinterpret_cast<AlzWindowArgs<kWinSmall>*>(blk));
  else fill(reinterpret_cast<AlzWindowArgs<kWinLarge>*>(blk));
}
