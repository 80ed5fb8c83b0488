// ptx.cuh -- carry-chain integer primitives for 256-bit modular arithmetic on sm_90a.
//
// On the device every primitive is exactly one PTX instruction; ptxas fuses each
// mad.lo.cc/madc.hi.cc pair into one IMAD.WIDE.U32(.X) with predicate carry (checked with
// cuobjdump -sass), so a 256-bit Montgomery product is ~136 IMAD-pipe instructions.
// Off the device (host pass of nvcc, or plain g++ for the CPU unit test of this header,
// tests/host/test_fp_host.cpp) the same names are emulated with an explicit carry flag so
// the field code above them can be validated bit-for-bit without a GPU.
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define CPB_HD __host__ __device__ __forceinline__
#define CPB_D __device__ __forceinline__
#else
#define CPB_HD inline
#define CPB_D inline
#endif

namespace cpb {

typedef uint32_t u32;
typedef uint64_t u64;

// Limb width.  32 on the device, always.  The host emulation below can be built with a narrower
// limb (tests/host/toy_field_shim.cpp: CPB_LIMB_BITS=8, a 64-bit "256-bit" field): every carry path
// of the algorithms in fp.cuh is then exercised by random operands (an all-ones limb is a 2^-8 event
// instead of 2^-32), which is how dropped carries are found.
#if !defined(CPB_LIMB_BITS) || defined(__CUDACC__)
#undef CPB_LIMB_BITS
#define CPB_LIMB_BITS 32
#endif
constexpr int LIMB_BITS = CPB_LIMB_BITS;
constexpr u32 LIMB_MASK = (u32)((1ull << CPB_LIMB_BITS) - 1);

#if defined(__CUDA_ARCH__)

CPB_D u32 mul_lo(u32 a, u32 b) { u32 r; asm("mul.lo.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
CPB_D u32 mul_hi(u32 a, u32 b) { u32 r; asm("mul.hi.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }

CPB_D u32 add_cc(u32 a, u32 b) { u32 r; asm volatile("add.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
CPB_D u32 addc_cc(u32 a, u32 b) { u32 r; asm volatile("addc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
CPB_D u32 addc(u32 a, u32 b) { u32 r; asm volatile("addc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
CPB_D u32 sub_cc(u32 a, u32 b) { u32 r; asm volatile("sub.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
CPB_D u32 subc_cc(u32 a, u32 b) { u32 r; asm volatile("subc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
CPB_D u32 subc(u32 a, u32 b) { u32 r; asm volatile("subc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }

// (lo,hi) += a*b as one 64-bit accumulate; the _cc forms start a chain, the c_ forms continue it.
CPB_D void mad_wide_cc(u32& lo, u32& hi, u32 a, u32 b) {
    asm volatile("mad.lo.cc.u32 %0, %2, %3, %0; madc.hi.cc.u32 %1, %2, %3, %1;" : "+r"(lo), "+r"(hi) : "r"(a), "r"(b));
}
CPB_D void madc_wide_cc(u32& lo, u32& hi, u32 a, u32 b) {
    asm volatile("madc.lo.cc.u32 %0, %2, %3, %0; madc.hi.cc.u32 %1, %2, %3, %1;" : "+r"(lo), "+r"(hi) : "r"(a), "r"(b));
}
// (lo,hi) = a*b + (c_lo,c_hi) + CF, continuing a chain (used for the 2-limb right shift).
CPB_D void madc_wide_cc_from(u32& lo, u32& hi, u32 a, u32 b, u32 c_lo, u32 c_hi) {
    asm volatile("madc.lo.cc.u32 %0, %2, %3, %4; madc.hi.cc.u32 %1, %2, %3, %5;"
                 : "=&r"(lo), "=r"(hi) : "r"(a), "r"(b), "r"(c_lo), "r"(c_hi));
}
// (lo,hi) = a*b + (c_lo,c_hi), starting a chain.
CPB_D void mad_wide_cc_from(u32& lo, u32& hi, u32 a, u32 b, u32 c_lo, u32 c_hi) {
    asm volatile("mad.lo.cc.u32 %0, %2, %3, %4; madc.hi.cc.u32 %1, %2, %3, %5;"
                 : "=&r"(lo), "=r"(hi) : "r"(a), "r"(b), "r"(c_lo), "r"(c_hi));
}
// (lo,hi) = a*b + CF; ends a chain (cannot overflow: a*b + 1 < 2^64).
CPB_D void madc_wide_end(u32& lo, u32& hi, u32 a, u32 b) {
    asm volatile("madc.lo.cc.u32 %0, %2, %3, 0; madc.hi.u32 %1, %2, %3, 0;" : "=&r"(lo), "=r"(hi) : "r"(a), "r"(b));
}
// (lo,hi) = a*b + c_lo + CF; ends a chain (a*b + 2 < 2^64 when c_lo <= 1: callers pass a carry word).
CPB_D void madc_wide_end_from(u32& lo, u32& hi, u32 a, u32 b, u32 c_lo) {
    asm volatile("madc.lo.cc.u32 %0, %2, %3, %4; madc.hi.u32 %1, %2, %3, 0;" : "=&r"(lo), "=r"(hi) : "r"(a), "r"(b), "r"(c_lo));
}
// (lo,hi) = a*b + (c_lo,c_hi) + CF; ends a chain (callers prove the sum below 2^64).
CPB_D void madc_wide_end_from(u32& lo, u32& hi, u32 a, u32 b, u32 c_lo, u32 c_hi) {
    asm volatile("madc.lo.cc.u32 %0, %2, %3, %4; madc.hi.u32 %1, %2, %3, %5;"
                 : "=&r"(lo), "=r"(hi) : "r"(a), "r"(b), "r"(c_lo), "r"(c_hi));
}
// (lo,hi) = a*b + c_lo; no carry in or out.
CPB_D void mad_wide_end_from(u32& lo, u32& hi, u32 a, u32 b, u32 c_lo) {
    asm volatile("mad.lo.cc.u32 %0, %2, %3, %4; madc.hi.u32 %1, %2, %3, 0;" : "=&r"(lo), "=r"(hi) : "r"(a), "r"(b), "r"(c_lo));
}
CPB_D void mul_wide(u32& lo, u32& hi, u32 a, u32 b) {
    asm("mul.lo.u32 %0, %2, %3; mul.hi.u32 %1, %2, %3;" : "=&r"(lo), "=r"(hi) : "r"(a), "r"(b));
}

#else  // ---- host emulation (bit-exact model of the PTX carry flag; limbs of LIMB_BITS bits) ----

namespace detail {
inline u32& cf() { static thread_local u32 f = 0; return f; }
constexpr int W = LIMB_BITS;
constexpr u64 M = LIMB_MASK;
inline u64 join(u32 lo, u32 hi) { return ((u64)hi << W) | lo; }
inline void split(unsigned __int128 s, u32& lo, u32& hi) { lo = (u32)((u64)s & M); hi = (u32)((u64)(s >> W) & M); }
}
inline u32 mul_lo(u32 a, u32 b) { return (u32)(((u64)a * b) & detail::M); }
inline u32 mul_hi(u32 a, u32 b) { return (u32)((((u64)a * b) >> detail::W) & detail::M); }
inline u32 add_cc(u32 a, u32 b) { u64 s = (u64)a + b; detail::cf() = (u32)(s >> detail::W); return (u32)(s & detail::M); }
inline u32 addc_cc(u32 a, u32 b) { u64 s = (u64)a + b + detail::cf(); detail::cf() = (u32)(s >> detail::W); return (u32)(s & detail::M); }
inline u32 addc(u32 a, u32 b) { return (u32)(((u64)a + b + detail::cf()) & detail::M); }
inline u32 sub_cc(u32 a, u32 b) { u64 d = (u64)a - b; detail::cf() = (u32)(d >> 63); return (u32)(d & detail::M); }
inline u32 subc_cc(u32 a, u32 b) { u64 d = (u64)a - b - detail::cf(); detail::cf() = (u32)(d >> 63); return (u32)(d & detail::M); }
inline u32 subc(u32 a, u32 b) { return (u32)(((u64)a - b - detail::cf()) & detail::M); }
inline void mad_wide_cc(u32& lo, u32& hi, u32 a, u32 b) {
    unsigned __int128 s = (unsigned __int128)detail::join(lo, hi) + (u64)a * b;
    detail::split(s, lo, hi); detail::cf() = (u32)(s >> (2 * detail::W));
}
inline void madc_wide_cc(u32& lo, u32& hi, u32 a, u32 b) {
    unsigned __int128 s = (unsigned __int128)detail::join(lo, hi) + (u64)a * b + detail::cf();
    detail::split(s, lo, hi); detail::cf() = (u32)(s >> (2 * detail::W));
}
inline void madc_wide_cc_from(u32& lo, u32& hi, u32 a, u32 b, u32 c_lo, u32 c_hi) {
    unsigned __int128 s = (unsigned __int128)detail::join(c_lo, c_hi) + (u64)a * b + detail::cf();
    detail::split(s, lo, hi); detail::cf() = (u32)(s >> (2 * detail::W));
}
inline void mad_wide_cc_from(u32& lo, u32& hi, u32 a, u32 b, u32 c_lo, u32 c_hi) {
    unsigned __int128 s = (unsigned __int128)detail::join(c_lo, c_hi) + (u64)a * b;
    detail::split(s, lo, hi); detail::cf() = (u32)(s >> (2 * detail::W));
}
inline void madc_wide_end(u32& lo, u32& hi, u32 a, u32 b) {
    unsigned __int128 s = (unsigned __int128)((u64)a * b) + detail::cf();
    detail::split(s, lo, hi);
}
inline void madc_wide_end_from(u32& lo, u32& hi, u32 a, u32 b, u32 c_lo) {
    unsigned __int128 s = (unsigned __int128)((u64)a * b) + c_lo + detail::cf();
    detail::split(s, lo, hi);
}
inline void madc_wide_end_from(u32& lo, u32& hi, u32 a, u32 b, u32 c_lo, u32 c_hi) {
    unsigned __int128 s = (unsigned __int128)detail::join(c_lo, c_hi) + (u64)a * b + detail::cf();
    detail::split(s, lo, hi);
}
inline void mad_wide_end_from(u32& lo, u32& hi, u32 a, u32 b, u32 c_lo) {
    unsigned __int128 s = (unsigned __int128)((u64)a * b) + c_lo;
    detail::split(s, lo, hi);
}
inline void mul_wide(u32& lo, u32& hi, u32 a, u32 b) { detail::split((unsigned __int128)((u64)a * b), lo, hi); }

#endif

}  // namespace cpb
