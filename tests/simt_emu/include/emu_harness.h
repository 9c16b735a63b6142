// What every SIMT-emulator harness (tests/simt_emu/<name>_emu.cpp) shares.  TEST INFRASTRUCTURE ONLY.
//
// tests/emu.py builds a harness two ways:
// - As a shared library the tests drive through ctypes.  Each request struct has a ctypes mirror in tests/emu.py, and
//   EMU_EXPORT_SIZEOF lets the loader compare the two layouts, so a field added on one side only fails at load time
//   instead of shifting every later pointer.
// - With -DRACE_<NAME> (the harness's name upper-cased: RACE_NUTS, RACE_DENSE_ADAPT, ...) as a program of its own, built
//   under ThreadSanitizer or AddressSanitizer.  Every CUDA thread is a host thread and the only synchronisation is what the
//   kernel itself asks for (shuffles / votes / __syncwarp -> the warp's barrier, __syncthreads -> the block's, mbarriers
//   and atomics -> std::atomic_ref), so a missing barrier or fence in the kernel is a data race TSan reports -- the CPU
//   counterpart of compute-sanitizer's racecheck, and it also covers the staged compile-time variants that have not run on
//   a GPU yet.  A harness that includes another one does not see that one's main: the macro names the harness built.
#pragma once
#include <cstddef>

// runs kernel(args) on blocks x threads emulated CUDA threads (simt_emu.cpp)
void emu_launch(void (*kernel)(const void*), const void* args, int blocks, int threads);

#define EMU_EXPORT_SIZEOF(T) \
    extern "C" size_t emu_sizeof_##T() { return sizeof(T); }
