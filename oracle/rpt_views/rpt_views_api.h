/* rpt_views_api.h -- entry points of librpt_views.so: the ReSTIR PT debug views (RPT_DEBUG_VIEW, IndirectLighting_Common.h:58-67)
 * restated on the CPU oracle's frame (test infrastructure, not product code).
 *
 * The oracle renders a frame as it does without a view (orc_rpt_render); a view changes only what the reference writes to FINAL at
 * three write points, so the view is applied afterwards, one write point at a time, from the planes that write point read:
 *   RPTV_PATHTRACE  ReSTIR_PT_PathTrace.hlsl:540-556 (temporal reuse off)
 *   RPTV_TTC        Reconnect_TtC.hlsl (temporal reuse without spatial reuse): the coloured write :386-388, the black early outs
 *   RPTV_STC        Reconnect_StC.hlsl, once per spatial pass: the coloured write :348-351, the black early outs
 * Plain C types only, parsed by zetaray_b200/_lib.prototypes like orc_api.h. */
#ifndef RPT_VIEWS_API_H
#define RPT_VIEWS_API_H

#include "../orc_api.h"

#ifdef __cplusplus
extern "C" {
#endif

#define RPTV_API __attribute__((visibility("default")))

/* RPT_Util::DebugColor (ReSTIR_PT/Util.hlsli:69-139) for view of the reconnection in meta[i] (a reservoir record's first word) over
 * the colour li[i] (3 floats) */
RPTV_API void rptv_debug_color(uint32_t view, const uint32_t* meta, const float* li, uint32_t n, float* out);

/* One write point of a frame the oracle rendered. For each pixel the write point's dispatch writes (its lanes through the group
 * swizzle and, with `sorted`, the thread map): black where the reference takes a WriteOutputColor early out, else DebugColor of
 * the reconnection in res_out; FINAL's rgb becomes that colour, or before's rgb plus it where the write point accumulates. res_gate:
 * the previous frame's reservoirs (RPTV_TTC) or the spatial pass's input reservoirs (RPTV_STC); neighbor: the pass's spatial
 * neighbours (RPTV_STC). final_img and before are float4 per pixel; final_img's alpha is left as it is. */
#define RPTV_PATHTRACE 0u
#define RPTV_TTC 1u
#define RPTV_STC 2u
RPTV_API void rptv_write_point(void* scene, const zr_frame_constants* fc, const uint32_t* core, const uint32_t* me, const uint32_t* coat,
    const uint32_t* pcore, const uint32_t* pcoat, uint32_t stage, uint32_t view, uint32_t sorted, const zr_rpt_reservoir* res_out,
    const zr_rpt_reservoir* res_gate, const uint16_t* neighbor, const uint16_t* thread_map, const float* before, float* final_img);

#ifdef __cplusplus
}
#endif

#endif
