// hostsim_io.cpp -- TEST INFRASTRUCTURE. Host (g++) build of the ReSTIR PT per-pixel I/O helpers (zetaray_b200/csrc/zr_rpt_io.cuh) and the
// storage codecs they rely on. A translation unit of its own: zr_rpt_io.cuh and zr_rgi.cuh reuse names in the library's unnamed namespace.
#include "prelude.h"
#include "hostsim_api.h"
#include "../../zetaray_b200/csrc/zr_rpt_io.cuh"

namespace zr
{
void set_error(const char*, ...) {}
}

// ---- "reservoir did not change" copy (zr_rpt_io.cuh CopyToNextFrame): the short cut that moves the reconnection words without
// decoding them against the decode + encode it replaces; out / ref stay zero for empty reservoirs (a partial write, not compared) ----
extern "C" void hostsim_probe_copy_to_next_frame(const zr_rpt_reservoir* in, uint32_t n, uint32_t M_max, zr_rpt_reservoir* out, zr_rpt_reservoir* ref,
    uint32_t* usedShortCut)
{
    uint32_t fast = 0;
    for (uint32_t i = 0; i < n; i++)
    {
        zr::RPT::Reservoir r = zr::RPT::Reservoir::Load_NonReconnection(in[i]);
        if (r.rc.Empty()) continue;
        zr::CopyToNextFrame(in[i], &out[i], r, M_max);
        zr::RPT::Reservoir r2 = zr::RPT::Reservoir::Load(in[i]);
        r2.Write(ref[i], M_max);
        fast += zr::RecordSurvivesRoundTrip(in[i]) ? 1u : 0u;
    }
    *usedShortCut = fast;
}
// EncodeOct32u(DecodeOct32(c)) over all 2^32 codes: returns how many codes with both halves strictly inside (0, 0xffff) change
extern "C" uint64_t hostsim_oct32_round_trip(int threads, uint64_t* boundaryChanged)
{
    std::atomic<uint64_t> bad{0}, badBoundary{0};
    std::atomic<uint32_t> next{0};
    auto work = [&]() {
        for (;;)
        {
            const uint32_t c = next.fetch_add(1);
            if (c >= 4096) break;
            uint64_t lb = 0, lbb = 0;
            for (uint64_t e = (uint64_t)c << 20; e < ((uint64_t)c + 1) << 20; e++)
            {
                const uint32_t code = (uint32_t)e, x = code & 0xffff, y = code >> 16;
                if (zr::Math::EncodeOct32u(zr::Math::DecodeOct32(code)) != code)
                {
                    if (x != 0 && x != 0xffff && y != 0 && y != 0xffff) lb++; else lbb++;
                }
            }
            bad += lb; badBoundary += lbb;
        }
    };
    std::vector<std::thread> th;
    for (int i = 0; i < (threads < 1 ? 1 : threads); i++) th.emplace_back(work);
    for (auto& t : th) t.join();
    if (boundaryChanged) *boundaryChanged = badBoundary.load();
    return bad.load();
}

