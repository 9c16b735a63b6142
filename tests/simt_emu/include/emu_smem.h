// The dynamic shared memory of an emulated launch (tests/simt_emu/simt_emu.cpp).  TEST INFRASTRUCTURE ONLY.
//
// On the device, shared memory holds whatever the previous block left there, and an access beyond the launch's allocation
// faults.  The emulator makes both visible on the CPU: a harness registers exactly the bytes the library's launcher asks
// for (the size functions next to the kernels), the emulator fills them and a guard zone on each side with a poison value
// before every block, checks after every block that the guards are untouched, and refuses a bulk copy or an mbarrier
// outside the registered bytes.  A kernel that reads padding it never wrote then computes with NaN (or +-1e300), and one
// that writes past its allocation is reported with the kernel, the block and the byte offset.
#pragma once
#include <cstddef>
#include <cstdint>

constexpr size_t kEmuSmemGuard = 64 * 1024;  // guard bytes on each side of the launch's shared memory
constexpr size_t kEmuSmemLimit = 232448;     // dynamic + static shared memory a block may have on sm_90 (227 KB)
constexpr size_t kEmuSmemArena = kEmuSmemGuard + kEmuSmemLimit + kEmuSmemGuard;
enum { EMU_POISON_NAN = 0, EMU_POISON_HUGE = 1 };  // a quiet NaN with a recognisable payload, or +-1e300 alternating

// the next launches' dynamic shared memory: [base, base + bytes), with kEmuSmemGuard bytes the caller owns on each side
// (an arena of kEmuSmemArena bytes, base = arena + kEmuSmemGuard); aborts if bytes + static_bytes exceed kEmuSmemLimit
void emu_smem_begin(unsigned char* base, size_t bytes, size_t static_bytes, const char* kernel);
void emu_smem_end();
bool emu_in_smem(const void* p, size_t bytes);
const char* emu_smem_kernel();
extern "C" void emu_set_poison(int mode);  // EMU_POISON_NAN (default) or EMU_POISON_HUGE
extern "C" int emu_get_poison();

// A kernel that declares `extern __shared__ double smem[]` resolves it to ahmc::smem.  This defines ahmc::smem as the
// usable part of an arena of the harness's translation unit (an assembler alias: the guard zone in front of it belongs to
// the same object, so an access below smem[0] lands in the guard instead of in some other variable).
#define EMU_DEFINE_SMEM_ARENA()                                                                      \
    namespace ahmc {                                                                                 \
    alignas(4096) unsigned char emu_smem_arena[kEmuSmemArena];                                       \
    }                                                                                                \
    asm(".globl _ZN4ahmc4smemE\n.set _ZN4ahmc4smemE, _ZN4ahmc14emu_smem_arenaE + 65536\n");         \
    static unsigned char* emu_smem_base() { return ahmc::emu_smem_arena + kEmuSmemGuard; }           \
    static_assert(kEmuSmemGuard == 65536, "the alias above spells out the guard size")
