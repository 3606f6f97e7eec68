// Thin C wrapper around the REFERENCE's own alias-table code (compiled from /root/reference by
// oracle/ref_alias/build.sh into oracle/_ref/libref_alias.so). Test infrastructure only: used to
// pin oracle/orc_alias.cpp against the reference and as bench.py's `--impl reference` arm.
//
// Wraps: ZetaCore/Math/Sampling.cpp:13-158 (AliasTable_Normalize/Build/SampleAliasTable),
//        ZetaCore/Math/Common.cpp:72-140 (KahanSum), ZetaCore/Utility/RNG.h:33-90.
#include "ref_alias_api.h"
#include <Math/Sampling.h>
#include <Math/Common.h>
#include <Utility/RNG.h>
#include <Utility/Span.h>
#include <cstdint>
#include <cstdlib>
#include <cstring>

using namespace ZetaRay;
using namespace ZetaRay::Math;
using namespace ZetaRay::Util;

extern "C"
{
    // weights: any alignment (the reference's result depends on it, SURVEY 8a-1)
    float ref_kahan_sum(const float* w, int64_t n)
    {
        return Math::KahanSum(Span<float>(w, (size_t)n));
    }

    void ref_alias_normalize(float* w, int64_t n)
    {
        Math::AliasTable_Normalize(MutableSpan<float>(w, (size_t)n));
    }

    // table: n x {P_Curr, P_Orig, Alias(u32)} (AliasTableEntry, Math/Sampling.h:18-23)
    void ref_alias_build(float* w, int64_t n, void* table)
    {
        AliasTableEntry* t = reinterpret_cast<AliasTableEntry*>(table);
        for (int64_t i = 0; i < n; i++)
            t[i] = AliasTableEntry{};
        Math::AliasTable_Build(MutableSpan<float>(w, (size_t)n), MutableSpan<AliasTableEntry>(t, (size_t)n));
    }

    void ref_alias_sample(const void* table, int64_t n, uint64_t stream_id, int num_draws,
        uint32_t* out_idx, float* out_pdf)
    {
        const AliasTableEntry* t = reinterpret_cast<const AliasTableEntry*>(table);
        RNG rng(stream_id);
        for (int i = 0; i < num_draws; i++)
        {
            float pdf;
            out_idx[i] = Math::SampleAliasTable(Span<AliasTableEntry>(t, (size_t)n), rng, pdf);
            out_pdf[i] = pdf;
        }
    }

    // first `count` outputs of Util::RNG(stream_id): uint then float alternately is not needed;
    // mode 0 = UniformUint, 1 = Uniform, 2 = UniformUintBounded(bound)
    void ref_rng_stream(uint64_t stream_id, int mode, uint32_t bound, int count, uint32_t* out_u, float* out_f)
    {
        RNG rng(stream_id);
        for (int i = 0; i < count; i++)
        {
            if (mode == 0) out_u[i] = rng.UniformUint();
            else if (mode == 1) out_f[i] = rng.Uniform();
            else out_u[i] = rng.UniformUintBounded(bound);
        }
    }

    float ref_halton(int i, int b)
    {
        return Math::Halton(i, b);
    }
}
