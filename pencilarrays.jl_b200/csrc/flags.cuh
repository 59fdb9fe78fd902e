// Flag words over NVLink, the device side of the one-sided protocols (kernels.cu: k_flags,
// k_multi; fft.cu: k_get_fft).
//
// A word only ever increases: signals are max-reductions with release semantics
// at system scope (every earlier store of this GPU, peer memory included, is
// visible before the new value), waits are acquire loads.  A wait that exceeds
// the time-out records the failure in mapped host memory and traps: nothing that
// depends on the missing peer may run on.
#pragma once

namespace pa {

__device__ __forceinline__ void flag_signal(unsigned long long* remote, unsigned long long seq) {
  __threadfence_system();
  asm volatile("red.release.sys.global.max.u64 [%0], %1;" ::"l"(remote), "l"(seq) : "memory");
}
__device__ __forceinline__ void flag_wait(const unsigned long long* local, unsigned long long seq,
                                          unsigned long long timeout_ns, int* err) {
  unsigned long long t0, now, v;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
  for (;;) {
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(local) : "memory");
    if (v >= seq) return;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
    if (timeout_ns && now - t0 > timeout_ns) {
      if (err) {
        *(volatile int*)err = 1;
        __threadfence_system();
      }
      __trap();
    }
    __nanosleep(100);
  }
}

}  // namespace pa
