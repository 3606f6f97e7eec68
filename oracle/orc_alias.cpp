// ORACLE -- test infrastructure, not product code (see orc_math.h header).
//
// CPU restatement of the reference's alias-table path (SURVEY 8a-1..a-4):
//   Math::KahanSum              ZetaCore/Math/Common.cpp:72-140   (8-lane AVX order restated in scalar code)
//   Math::AliasTable_Normalize  ZetaCore/Math/Sampling.cpp:13-50
//   Math::AliasTable_Build      ZetaCore/Math/Sampling.cpp:52-143 (tested twin)
//   BuildAliasTable             ZetaRenderPass/PreLighting/PreLighting.cpp:27-158 (production)
//   Math::SampleAliasTable      ZetaCore/Math/Sampling.cpp:145-158
//   Util::RNG                   ZetaCore/Utility/RNG.h:33-90 (PCG-XSH-RR 64->32)
//   Light::AliasTableSample     ZetaRenderPass/Common/LightSource.hlsli:72-97 (GPU twin, 32-bit PCG)
//   Math::Halton                ZetaCore/Math/Sampling.cpp:160-174
// Pinned against the reference itself (oracle/_ref/libref_alias.so) and the golden vector of
// SURVEY 8c by tests/test_alias_oracle.py.
#include "orc_api.h"
#include "orc_math.h"
#include <vector>
#include <cstdlib>

using namespace orc;

namespace
{
    struct KahanAcc
    {
        float sum = 0.0f;
        float compensation = 0.0f;
        void add(float v)
        {
            float corrected = v - compensation;
            float newSum = sum + corrected;
            compensation = (newSum - sum) - corrected;
            sum = newSum;
        }
    };

    // Util::RNG
    struct RNG64
    {
        uint64_t State, Inc;
        explicit RNG64(uint64_t streamID)
        {
            State = 0U;
            Inc = (streamID << 1u) | 1u;
            UniformUint();
            State += 0x853c49e6748fea9bULL;
            UniformUint();
        }
        uint32_t UniformUint()
        {
            uint64_t oldstate = State;
            State = oldstate * 6364136223846793005ULL + Inc;
            uint32_t xorshifted = (uint32_t)(((oldstate >> 18u) ^ oldstate) >> 27u);
            uint32_t rot = (uint32_t)(oldstate >> 59u);
            return (xorshifted >> rot) | (xorshifted << ((~rot + 1u) & 31));
        }
        float Uniform() { return float(UniformUint() >> 8) * 0x1p-24f; }
        uint32_t UniformUintBounded(uint32_t bound)
        {
            uint32_t threshold = (~bound + 1u) % bound;
            for (;;)
            {
                uint32_t r = UniformUint();
                if (r >= threshold)
                    return r % bound;
            }
        }
    };
}

extern "C"
{
    // `prologue` = number of leading elements the reference would add one by one before reaching a
    // 32-byte boundary ((32 - addr % 32) / 4 % 8 for a 4-byte aligned pointer; 0 in production).
    float orc_kahan_sum(const float* data, int64_t N, int prologue)
    {
        KahanAcc acc;
        int64_t start = prologue < N ? prologue : N;
        for (int64_t i = 0; i < start; i++)
            acc.add(data[i]);

        int64_t numSIMD = N - start;
        numSIMD -= numSIMD & 15;
        float vSum[8] = { 0 }, vComp[8] = { 0 };
        for (int64_t i = start; i < start + numSIMD; i += 16)
        {
            for (int l = 0; l < 8; l++)
            {
                float vCurr = data[i + l] + data[i + 8 + l];
                float vCorrected = vCurr - vComp[l];
                float vNewSum = vSum[l] + vCorrected;
                float c = vNewSum - vSum[l];
                vComp[l] = c - vCorrected;
                vSum[l] = vNewSum;
            }
        }
        for (int l = 0; l < 8; l++)
        {
            float corrected = vSum[l] - acc.compensation - vComp[l];
            float newSum = acc.sum + corrected;
            acc.compensation = (newSum - acc.sum) - corrected;
            acc.sum = newSum;
        }
        for (int64_t i = start + numSIMD; i < N; i++)
            acc.add(data[i]);
        return acc.sum;
    }

    void orc_alias_normalize(float* w, int64_t N, int prologue)
    {
        const float sum = orc_kahan_sum(w, N, prologue);
        const float sumRcp = (float)N / sum;
        for (int64_t i = 0; i < N; i++)
            w[i] *= sumRcp;
    }

    // Vose's method with LIFO stacks, indices pushed in index order. out: P_Curr, P_Orig, Alias per entry.
    static void vose(float* probs, int64_t N, float* P_Curr, uint32_t* Alias)
    {
        std::vector<uint32_t> larger, smaller;
        larger.reserve((size_t)N);
        smaller.reserve((size_t)N);
        for (int64_t i = 0; i < N; i++)
        {
            if (probs[i] < 1.0f) smaller.push_back((uint32_t)i);
            else larger.push_back((uint32_t)i);
        }
        while (!smaller.empty() && !larger.empty())
        {
            const uint32_t smallerIdx = smaller.back();
            smaller.pop_back();
            const float smallerProb = probs[smallerIdx];
            const uint32_t largerIdx = larger.back();
            float largerProb = probs[largerIdx];
            Alias[smallerIdx] = largerIdx;
            P_Curr[smallerIdx] = smallerProb;
            largerProb = (smallerProb + largerProb) - 1.0f;
            probs[largerIdx] = largerProb;
            if (largerProb < 1.0f)
            {
                larger.pop_back();
                smaller.push_back(largerIdx);
            }
        }
        while (!larger.empty())
        {
            uint32_t idx = larger.back(); larger.pop_back();
            Alias[idx] = idx; P_Curr[idx] = 1.0f;
        }
        while (!smaller.empty())
        {
            uint32_t idx = smaller.back(); smaller.pop_back();
            Alias[idx] = idx; P_Curr[idx] = 1.0f;
        }
    }

    // Tested twin: table = N x {P_Curr, P_Orig, Alias}
    void orc_alias_build(float* probs, int64_t N, int prologue, void* table_)
    {
        struct E { float P_Curr, P_Orig; uint32_t Alias; };
        E* table = (E*)table_;
        const float oneDivN = 1.0f / (float)N;
        orc_alias_normalize(probs, N, prologue);
        std::vector<float> pc((size_t)N);
        std::vector<uint32_t> al((size_t)N);
        for (int64_t i = 0; i < N; i++)
            table[i].P_Orig = probs[i] * oneDivN;
        vose(probs, N, pc.data(), al.data());
        for (int64_t i = 0; i < N; i++) { table[i].P_Curr = pc[i]; table[i].Alias = al[i]; }
    }

    // Production: table = N x {CachedP_Orig, CachedP_Alias, P_Curr, Alias}
    void orc_alias_build_emissive(float* probs, int64_t N, int prologue, void* table_)
    {
        struct E { float CachedP_Orig, CachedP_Alias, P_Curr; uint32_t Alias; };
        E* table = (E*)table_;
        const float oneDivN = 1.0f / (float)N;
        orc_alias_normalize(probs, N, prologue);
        std::vector<float> pc((size_t)N);
        std::vector<uint32_t> al((size_t)N);
        for (int64_t i = 0; i < N; i++)
            table[i].CachedP_Orig = probs[i] * oneDivN;
        vose(probs, N, pc.data(), al.data());
        for (int64_t i = 0; i < N; i++) { table[i].P_Curr = pc[i]; table[i].Alias = al[i]; }
        for (int64_t i = 0; i < N; i++)
            table[i].CachedP_Alias = table[table[i].Alias].CachedP_Orig;
    }

    void orc_alias_sample(const void* table_, int64_t N, uint64_t stream_id, int num_draws,
        uint32_t* out_idx, float* out_pdf)
    {
        struct E { float P_Curr, P_Orig; uint32_t Alias; };
        const E* table = (const E*)table_;
        RNG64 rng(stream_id);
        for (int i = 0; i < num_draws; i++)
        {
            uint32_t idx = rng.UniformUintBounded((uint32_t)N);
            E s = table[idx];
            if (rng.Uniform() < s.P_Curr) { out_pdf[i] = s.P_Orig; out_idx[i] = idx; }
            else { out_pdf[i] = table[s.Alias].P_Orig; out_idx[i] = s.Alias; }
        }
    }

    void orc_rng64_stream(uint64_t stream_id, int mode, uint32_t bound, int count, uint32_t* out_u, float* out_f)
    {
        RNG64 rng(stream_id);
        for (int i = 0; i < count; i++)
        {
            if (mode == 0) out_u[i] = rng.UniformUint();
            else if (mode == 1) out_f[i] = rng.Uniform();
            else out_u[i] = rng.UniformUintBounded(bound);
        }
    }

    // GPU twin with the shader RNG: consecutive draws of RNG::Init(seed)
    void orc_alias_sample_gpu(const void* table_, uint32_t N, uint32_t seed, uint32_t num_draws,
        uint32_t* out_idx, float* out_pdf)
    {
        struct E { float CachedP_Orig, CachedP_Alias, P_Curr; uint32_t Alias; };
        const E* table = (const E*)table_;
        RNG rng = RNG::InitSeed(seed);
        for (uint32_t i = 0; i < num_draws; i++)
        {
            uint32_t u0 = rng.UniformUintBounded(N);
            E s = table[u0];
            if (rng.Uniform() < s.P_Curr) { out_pdf[i] = s.CachedP_Orig; out_idx[i] = u0; }
            else { out_pdf[i] = s.CachedP_Alias; out_idx[i] = s.Alias; }
        }
    }

    float orc_halton(int i, int b)
    {
        float f = 1.0f, r = 0.0f, bf = (float)b;
        while (i > 0)
        {
            f /= bf;
            r = r + f * (float)(i % b);
            i = (int)((float)i / bf);
        }
        return r;
    }

    // shader hashes for integer-exact tests
    void orc_pcg3d(uint32_t x, uint32_t y, uint32_t z, uint32_t out[3])
    {
        uint3 v = RNG::PCG3d(uint3{ x, y, z }); out[0] = v.x; out[1] = v.y; out[2] = v.z;
    }
    void orc_pcg4d(uint32_t x, uint32_t y, uint32_t z, uint32_t w, uint32_t out[4])
    {
        uint4 v = RNG::PCG4d(uint4{ x, y, z, w }); out[0] = v.x; out[1] = v.y; out[2] = v.z; out[3] = v.w;
    }
    uint32_t orc_pcg(uint32_t x) { return RNG::PCG(x); }
    void orc_rng32_stream(uint32_t seed, int count, uint32_t* out_u, float* out_f)
    {
        RNG rng = RNG::InitSeed(seed);
        for (int i = 0; i < count; i++) { uint32_t s = rng.State; RNG t = RNG::InitSeed(s); out_f[i] = t.Uniform(); out_u[i] = rng.UniformUint(); }
    }
}
