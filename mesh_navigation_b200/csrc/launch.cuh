// Launch / dynamic-shared-memory macros shared by the kernel headers and the host code.
#pragma once
// Kernel launches go through one macro: the CPU interpreter behind the `-m "not gpu"` logic tests (tests/emu/) compiles
// this very file with g++, which has no <<<>>>.  MNB_EMU_ACTIVE is only ever defined by tests/emu/cuda_runtime.h; the
// shipped library is built by nvcc without it and contains no host execution path for any kernel.
#ifdef MNB_EMU_ACTIVE
// <<<>>> converts the arguments to the kernel's parameter types (a DeviceBuffer to its pointer); the interpreter's launch
// takes them as given, so they are converted here
template <class... KArgs, class... Args>
static inline cudaError_t mnb_interpreted_launch(void (*kern)(KArgs...), unsigned grid, unsigned block, size_t smem, Args&&... args) {
  return emu::launch(kern, grid, block, smem, 1u, false, static_cast<std::decay_t<KArgs>>(std::forward<Args>(args))...);
}
#define MNB_LAUNCH(kern, grid, block, smem, stream, ...) \
  mnb_interpreted_launch(kern, (unsigned)(grid), (unsigned)(block), (size_t)(smem), __VA_ARGS__)
#define MNB_DYNAMIC_SMEM(name) unsigned char* name = emu::g_cta.dyn_smem
#else
#define MNB_LAUNCH(kern, grid, block, smem, stream, ...) kern<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__)
#define MNB_DYNAMIC_SMEM(name) extern __shared__ __align__(16) unsigned char name[]
#endif

// fire-and-forget prefetch of the line at p into the L2 (no register, no scoreboard); a no-op on the CPU interpreter
#ifdef MNB_EMU_ACTIVE
static inline void mnb_prefetch_l2(const void*) {}
#else
__device__ __forceinline__ void mnb_prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
#endif
