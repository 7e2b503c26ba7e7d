// TEST INFRASTRUCTURE ONLY -- storage for the emulated builtin index variables and the failure hook.
#include "cuda_runtime.h"
thread_local emuIdx threadIdx, blockIdx, blockDim, gridDim;
thread_local EmuWarpSync *emu_warp = nullptr;
thread_local EmuBlockSync *emu_block = nullptr;
thread_local unsigned char *emu_smem = nullptr;
std::atomic<int> emu_fail_in{0};
std::atomic<long> emu_live_allocs{0};

// the failure hook of the emulation library only (tests/test_host_entries.py binds them itself)
extern "C" __attribute__((visibility("default"))) void sb_emu_fail_at(int k) { emu_fail_in = k; }
extern "C" __attribute__((visibility("default"))) long sb_emu_live_allocs(void) { return emu_live_allocs.load(); }
