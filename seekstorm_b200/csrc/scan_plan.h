// scan_plan.h — which vector scan a search runs (DESIGN.md §3.2).  Host code without CUDA: g++ compiles it on its own.
#pragma once
#include <stdint.h>

#include "../../include/seekstorm_b200.h"

namespace ssb {
namespace vec {

// one value per launchable scan: kernel, operand precision and queries per corpus pass
enum class Scan { Ffma, Tf32_64, Tf32_128, Bf16_64, Bf16_128, Bf16_256, I8_128, F16f_128, F16f_256, F16f_256Pair };

constexpr uint32_t queries_per_pass(Scan s) {
    return s == Scan::Ffma ? 16 : (s == Scan::Tf32_64 || s == Scan::Bf16_64) ? 64 : (s == Scan::Bf16_256 || s == Scan::F16f_256 || s == Scan::F16f_256Pair) ? 256 : 128;
}
// the filter scan (DESIGN.md §3.2c): one fp16 product selects <= 32 candidates per query, refine_candidates re-scores them in f32
constexpr bool is_filter(Scan s) { return s == Scan::F16f_128 || s == Scan::F16f_256 || s == Scan::F16f_256Pair; }
constexpr bool is_tensor_core(Scan s) { return s != Scan::Ffma; }

// kernel: SSB_VEC_KERNEL_* (ssb_create and ssb_set_vector_kernel reject anything above 9); has_f16_plane: the index holds the filter
// scan's fp16 plane and its error bounds; paging: the call passes key ceilings (pages beyond the first 32 results).
// AUTO (measured on one H100 SXM, 700 W, 1M x 768): one FP32 pass of 16 queries takes ~0.97 ms, one 3xBF16 tensor-core pass of up
// to 128 queries ~1.08 ms -> FP32 scan for <= 16 queries, tensor-core scan above.  The filter scan + exact refine (DESIGN.md §3.2c)
// reads half the bytes and does a third of the tensor work per pass, so AUTO takes it at every batch size when it can run: one
// 128-query filter pass (0.59 ms on 1M x 768) also beats the FP32 scan's 0.97 ms pass for <= 16 queries, and above 128 queries one
// 256-query pass (0.88 ms, measured; 1.2 ms on CTA pairs) beats two 128-query passes (1.17-1.20 ms).
inline Scan plan_scan(uint32_t kernel, uint32_t similarity, bool quant_i8, bool has_f16_plane, uint32_t nq, uint32_t k, bool paging) {
    if (quant_i8) return Scan::I8_128;                        // one kernel for the int8 corpus: s8 wgmma, 128-query tile
    if (similarity == SSB_SIM_EUCLIDEAN) return Scan::Ffma;   // the f32 tensor-core scans score Dot / Cosine only
    // the filter scan keeps a candidate set sized for k <= 16 in the 32-entry lists and has no paging (ceilings are exact keys)
    const bool filterable = k <= 16 && !paging && has_f16_plane;
    // the exact 3xBF16 scan takes the 256-query tile (2.37 ms per pass vs 1.08 ms for 128 queries, measured) when it needs fewer
    // milliseconds for this batch: ceil(nq/256) * 2.37 < ceil(nq/128) * 1.08 (with these figures it never does: 2.37 > 2 * 1.08)
    const Scan exact = (nq + 255u) / 256u * 237u < (nq + 127u) / 128u * 108u ? Scan::Bf16_256 : Scan::Bf16_128;
    switch (kernel) {
    case SSB_VEC_KERNEL_AUTO: return filterable ? (nq <= 128 ? Scan::F16f_128 : Scan::F16f_256) : (nq <= 16 ? Scan::Ffma : exact);
    case SSB_VEC_KERNEL_FFMA: return Scan::Ffma;
    case SSB_VEC_KERNEL_TCGEN05: return Scan::Tf32_128;
    case SSB_VEC_KERNEL_TCGEN05_N64: return Scan::Tf32_64;
    case SSB_VEC_KERNEL_TCGEN05_BF16: return Scan::Bf16_128;
    case SSB_VEC_KERNEL_TCGEN05_BF16_N64: return Scan::Bf16_64;
    case SSB_VEC_KERNEL_TCGEN05_BF16_N256: return Scan::Bf16_256;
    case SSB_VEC_KERNEL_TCGEN05_FILTER: return filterable ? Scan::F16f_128 : Scan::Bf16_128;
    case SSB_VEC_KERNEL_TCGEN05_FILTER_N256: return filterable ? Scan::F16f_256 : exact;
    default: return filterable ? Scan::F16f_256Pair : exact;   // SSB_VEC_KERNEL_TCGEN05_FILTER_N256_PAIR
    }
}

}  // namespace vec
}  // namespace ssb
