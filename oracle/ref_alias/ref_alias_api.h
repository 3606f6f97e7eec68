/* ref_alias_api.h -- the entry points of oracle/_ref/libref_alias.so (ref_alias_wrap.cpp around the reference's alias table,
 * KahanSum, RNG and Halton). Plain C types only: tests/orc.py binds each function's ctypes types from these prototypes, and the
 * wrapper includes this header, so a definition whose types differ from its declaration does not compile. */
#ifndef REF_ALIAS_API_H
#define REF_ALIAS_API_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define REF_API __attribute__((visibility("default")))

REF_API float ref_kahan_sum(const float* w, int64_t n);
REF_API void ref_alias_normalize(float* w, int64_t n);
/* table: n x {P_Curr, P_Orig, Alias(u32)} (AliasTableEntry) */
REF_API void ref_alias_build(float* w, int64_t n, void* table);
REF_API void ref_alias_sample(const void* table, int64_t n, uint64_t stream_id, int num_draws, uint32_t* out_idx, float* out_pdf);
/* mode 0 = UniformUint, 1 = Uniform, 2 = UniformUintBounded(bound) */
REF_API void ref_rng_stream(uint64_t stream_id, int mode, uint32_t bound, int count, uint32_t* out_u, float* out_f);
REF_API float ref_halton(int i, int b);

#ifdef __cplusplus
}
#endif

#endif
