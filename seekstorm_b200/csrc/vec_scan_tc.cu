// vec_scan_tc.cu — tensor-core variant of the brute-force vector scan (sm_90a: wgmma + TMA + mbarrier, thread-block clusters).
//
// Same contract as scan_ffma (vec_scan.cu): corpus [n_rows, Dpad] f32 x a block of NQ queries -> per-warp top-32 lists, but the
// query x corpus contraction runs on the Hopper tensor cores (warpgroup MMA, both operands in shared memory, accumulators in registers):
//   D[64 corpus rows, NQ/2 queries] (f32) += A[64 x K] . B[NQ/2 x K]^T          wgmma.mma_async.m64nNk*
// f32-level accuracy (north-star tolerance 1e-4 on cosine scores) comes from a 3-product split
//   a.b ~= a_hi.b_hi + a_lo.b_hi + a_hi.b_lo                (the dropped a_lo.b_lo term is second order)
// in one of two operand precisions, or exactly on int8 codes (template PREC):
//   PREC_TF32 : tf32 operands, x_hi = x & 0xFFFFE000 (exactly representable in tf32, so the result does not depend on
//               whether the tensor core truncates or rounds), x_lo = x - x_hi (exact); error ~2^-22 per product.
//   PREC_BF16 : bf16 operands, f32 accumulate, x_hi = bf16_rn(x), x_lo = bf16_rn(x - x_hi);
//               error ~3*2^-17 per product (random sign) -> ~1e-5 relative on a 768-d score.  Twice the MACs per MMA
//               instruction and half the operand bytes per MAC of tf32: the faster split.
//   PREC_I8   : s8 x s8 -> s32 over an int8 corpus (Cosine + ScalarQuantizationI8, quantised at load time): ONE exact product; the
//               TMA'd tile is the MMA operand (no splitting), the 128-query block stays resident in smem (template BRES) when it
//               leaves room for 3 corpus stages.  See DESIGN.md §3.2b.
// The query parts are prepared once per batch in global memory.  PREC_BF16: the corpus parts are prepared ONCE AT LOAD TIME as
// two bf16 planes (hi, lo) — together 4 bytes per element, so the algorithmic bytes of a pass stay n_rows*dims*4 — and TMA
// delivers them straight into the MMA-ready SWIZZLE_64B tiles: no splitting pass over the tile in shared memory.  PREC_TF32 keeps
// the f32 corpus and splits each stage in shared memory (out of place for the lo part).
//
// Warp roles (384 threads = 3 warpgroups, 1 CTA/SM): warpgroup 0 = TMA producer (one thread; 256 queries: + 3 list warps), warpgroups 1-2 = consumers.  Consumer
// warpgroup c owns the query columns [c*NQ/2, (c+1)*NQ/2) of the block and all TROWS corpus rows of a tile (TROWS/64 m64 sub-tiles,
// at most 128 accumulator registers per thread); warp w of the warpgroup owns rows 16w..16w+15 of every sub-tile and (64/128 queries)
// list w of the warpgroup's queries, so each (list, query) pair has exactly one writer, as in the scratch layout [4 lists][NQ][32] per CTA.
// Per stage both consumer warpgroups wait on the full barrier, issue their MMAs as one commit group (one group kept in flight) and
// release the stage once its group retired.  Epilogue per tile (the producer keeps streaming up to STAGES stages ahead meanwhile):
// the accumulator fragment goes 8 query columns at a time through a small per-warp shared-memory buffer into a lane = corpus row
// layout (one pass = 32 rows = two sub-tiles); the whole chunk is tested against the per-query thresholds branch-free with ONE vote,
// and only chunks with a candidate take the per-column path (ballot, per-warp sorted lists in the CTA's slice of the output scratch,
// no CTA barriers).  The 256-query kernels take that vote on the fragment itself, before the transposition, so that a chunk without
// a candidate costs no shared-memory traffic.  When the scan is seeded they do no list work in the consumer warps: a chunk that passes is written as a
// record into a shared-memory queue, and warps 1-3 of warpgroup 0 (idle otherwise: one thread issues the TMA loads) run the exact test
// and the inserts into one list per query per CTA ([NQ][32]), each warp for a fixed third of the 8-query chunks.  An insert is ~1 us of
// latency-bound work; in the consumer warps it held both warpgroups, and with them the tensor pipe, at the end of every tile.
// Threshold seeding: the same kernel runs first in sample mode over a few tiles per SM and writes per-(32-row group, query) score
// maxima (256 queries: reduced on the accumulator fragment by shuffles, without the transposition); kth_from_groupmax turns them into
// valid lower bounds of the k-th best score.  A seeded 256-query filter scan leaves its lists unmerged: refine_candidates merges them.
#include <cuda_bf16.h>
#include <stdlib.h>
#include <type_traits>
#include <cuda_fp16.h>

#include "common.cuh"
#include "vec_scan.h"

namespace ssb {
namespace vec {

namespace tc {
constexpr int KC = 32;                 // floats per k-chunk = one 128-byte swizzle row of the f32 corpus tile
constexpr int TM = 128;                // corpus rows per TMA tile unit
constexpr int MT = 2;                  // tile units per stage (128-query variants): the query chunk is fetched once per MT*128 corpus rows
constexpr int TROWS = TM * MT;         // corpus rows per stage
constexpr int A1_BYTES = TM * KC * 4;  // one 128-row f32 tile, 16 KB
constexpr int THREADS = 384;           // 3 warpgroups: TMA producer, 2 MMA + epilogue
constexpr int CHUNK = 8;               // query columns per epilogue step
constexpr int XB_STRIDE = CHUNK + 1;   // per-warp transposition buffer [32 rows][CHUNK] (+1 column: conflict-free row reads)
constexpr int REC_WORDS = 32 * XB_STRIDE;     // one warp's buffer: 32 rows x CHUNK scores
constexpr int XB_BYTES = 8 * REC_WORDS * 4;
// QUEUE kernels (seeded 256-query scans): the buffers form a queue of chunk records (one chunk = 32 rows x 8 queries that passed the
// vote) from the consumer warps to the list warps, plus per slot a state word (0 free, 1 being written, 2 + chunk = ready) and the
// record's (tile, warp), and a count of finished consumer warps.  26 slots keep the 256-query configurations at 4 stages.
constexpr int QSLOTS = 26;
constexpr int QUEUE_BYTES = QSLOTS * REC_WORDS * 4 + (3 * QSLOTS + 2) * 4;
constexpr int SMEM_MAX = 232448;       // 227 KB opt-in limit per CTA
constexpr uint32_t ORD_NEG_INF = 0x007FFFFFu;   // ord_f32(-inf)
enum { PREC_TF32 = 0, PREC_BF16 = 1, PREC_I8 = 2, PREC_F16F = 3 };
// PREC_F16F — the FILTER scan (DESIGN.md §3.2c): ONE product h(a).h(b) over an fp16 plane of the corpus (2 bytes per element, a third of
// the tensor work of the 3-product split; fp16 keeps 11 significand bits, bf16 8 — the margin below is 8x tighter than with the bf16
// hi plane; rows and queries are pre-scaled by powers of two into fp16's range, everything below lives in that scaled space and is
// never returned).  The approximate score s^ differs from the (scaled) f32 score s by at most eps_q =
// max_r|a_r - h(a_r)| * |b| + max_r|h(a_r)| * |b - h(b)| + accumulation slack (Cauchy-Schwarz; both row maxima are computed at load time),
// so every row of the exact top-k satisfies s^ >= (k-th best s^) - 2 eps_q.  The epilogue keeps exactly that candidate set (keys carry
// the ROW index, thresholds are lowered by the per-query margin 2 eps_q), refine_candidates (vec_refine.cu) re-scores the <= 32 candidates
// in f32 from the f32 rows and flags the queries whose candidate set may not have fitted the 32-entry list for the exact fallback scan.
// PAIR (filter scan, 256 queries): clusters of 2 CTAs on neighbouring corpus tiles share ONE copy of the query block: each CTA loads
// half of it per stage with TMA multicast into both CTAs' shared memory, so an SM takes in its corpus tile plus half a query block per
// stage instead of a whole one, and a stage is refilled once the consumers of BOTH CTAs released it.

constexpr int MAX_STAGES = 6;
template <int NQ, int PREC, bool BRES = false, bool QUEUE = false> struct Cfg {
    // at most 128 accumulator registers per consumer thread (TROWS/64 sub-tiles x NQ/4): 256 queries -> one 128-row tile per stage (the
    // corpus is streamed once per 256 queries: half the HBM bytes per query); tf32 -> 128 rows too (its stage also holds the lo part)
    static constexpr int MT = (NQ == 256 || PREC == PREC_TF32) ? 1 : 2;
    static constexpr int TROWS = TM * MT;
    static constexpr int MW = TROWS / 64;      // m64 sub-tiles per consumer warpgroup
    static constexpr int NQH = NQ / 2;         // query columns per consumer warpgroup = the MMA's N
    static constexpr int A_BYTES = MT * A1_BYTES;
    // TF32: [A (-> A_hi in place) | A_lo | B_hi | B_lo], all f32 SWIZZLE_128B tiles
    // BF16: [A1 bf16 (hi plane) | A2 bf16 (lo plane) | B1 bf16 | B2 bf16], 64-byte rows, SWIZZLE_64B, all four delivered by TMA.
    // I8  : [A i8 | B i8]: the int8 corpus (quantised at load time) is the MMA operand as TMA delivers it, 128 dims per 128-byte swizzle row
    // F16F: [A f16 | B f16], 64 halves per 128-byte swizzle row
    static constexpr int KCE = PREC == PREC_I8 ? 128 : (PREC == PREC_F16F ? 64 : KC);   // elements per k-chunk
    static constexpr int B_BYTES = PREC == PREC_BF16 ? NQ * KC * 2 : NQ * KC * 4;
    static constexpr int B_ROW = PREC == PREC_BF16 ? 64 : 128;                 // bytes per query row of a B tile
    static constexpr int ALO_OFF = PREC == PREC_BF16 ? 0 : A_BYTES;            // TF32: A_lo   | BF16: A1 (in place)
    static constexpr int A2_OFF = A_BYTES / 2;                                 // BF16: A2 (in place)
    static constexpr int B_OFF = PREC == PREC_TF32 ? 2 * A_BYTES : A_BYTES;
    // BRES (int8 only): the whole quantised query block [n_kchunks][NQ x 128 B] stays resident in smem behind the A stages,
    // so the per-stage L2->SM traffic is the corpus tile alone (stage count chosen at launch from what is left of 227 KB)
    static constexpr int STAGE_BYTES = BRES ? A_BYTES : ((PREC == PREC_I8 || PREC == PREC_F16F) ? A_BYTES + B_BYTES : (PREC == PREC_BF16 ? A_BYTES + 2 * B_BYTES : 2 * A_BYTES + 2 * B_BYTES));
    static constexpr int TX_BYTES = BRES ? A_BYTES : ((PREC == PREC_I8 || PREC == PREC_F16F) ? A_BYTES + B_BYTES : A_BYTES + 2 * B_BYTES);
    // transposition buffers (QUEUE: the record queue) + thresholds + (scaled int8) per-query scale / norm + barriers + alignment
    // slack of the dynamic segment
    static constexpr int XB_REGION = QUEUE ? QUEUE_BYTES : XB_BYTES;
    static constexpr int FIXED = XB_REGION + NQ * 12 + 256 + 1024;
    static constexpr int STAGES = (SMEM_MAX - FIXED) / STAGE_BYTES > MAX_STAGES ? MAX_STAGES : (SMEM_MAX - FIXED) / STAGE_BYTES;
    static constexpr int SMEM = STAGES * STAGE_BYTES + FIXED;
    static_assert(!QUEUE || (NQ == 256 && !BRES && STAGES >= 4), "the record queue is for the 256-query kernels and must leave them 4 stages");
    // a record names its rows by (tile, consumer warp): one pair of m64 sub-tiles per tile
    static_assert(!QUEUE || MW == 2, "queue records hold the one 32-row pass of a 128-row tile");
};
// int8: the query block stays resident when it leaves room for 3 corpus stages
constexpr bool i8_resident(uint32_t dpad8) { return (int)dpad8 * 128 + Cfg<128, PREC_I8, true>::FIXED + 3 * Cfg<128, PREC_I8, true>::A_BYTES <= SMEM_MAX; }

// wgmma shared-memory matrix descriptor for K-major swizzled tiles: start address >> 4 (bits 0-13), leading byte offset (unused by
// swizzled K-major layouts: 1), stride byte offset = one 8-row swizzle atom >> 4 (bits 32-45), swizzle mode (bits 62-63).
// SWIZZLE_128B: 128-byte rows, 1024-byte atom, mode 1
__device__ __forceinline__ uint64_t gmma_desc_k128(uint32_t saddr) {
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}
// SWIZZLE_64B: 64-byte rows, 512-byte atom, mode 2
__device__ __forceinline__ uint64_t gmma_desc_k64(uint32_t saddr) {
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | (1ull << 16) | (32ull << 32) | (2ull << 62);
}

// wgmma.mma_async m64nNk*, D (+)= A . B^T with both operands K-major in shared memory; acc = 0 overwrites D (first product of a tile)
__device__ __forceinline__ void wgmma_tf32_n32(float (&d)[16], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
                 "%16, %17, p, 1, 1;\n}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                 : "l"(a), "l"(b), "r"(acc) : "memory");
}
__device__ __forceinline__ void wgmma_tf32_n64(float (&d)[32], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
                 "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
                 "%32, %33, p, 1, 1;\n}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
                   "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "l"(a), "l"(b), "r"(acc) : "memory");
}
__device__ __forceinline__ void wgmma_bf16_n32(float (&d)[16], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
                 "%16, %17, p, 1, 1, 0, 0;\n}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                 : "l"(a), "l"(b), "r"(acc) : "memory");
}
__device__ __forceinline__ void wgmma_bf16_n64(float (&d)[32], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
                 "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
                 "%32, %33, p, 1, 1, 0, 0;\n}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
                   "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "l"(a), "l"(b), "r"(acc) : "memory");
}
__device__ __forceinline__ void wgmma_bf16_n128(float (&d)[64], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
                 "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31,"
                 "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47,"
                 "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
                 "%64, %65, p, 1, 1, 0, 0;\n}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
                   "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
                   "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
                   "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
                   "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
                   "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "l"(a), "l"(b), "r"(acc) : "memory");
}
__device__ __forceinline__ void wgmma_f16_n64(float (&d)[32], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
                 "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
                 "%32, %33, p, 1, 1, 0, 0;\n}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
                   "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "l"(a), "l"(b), "r"(acc) : "memory");
}
__device__ __forceinline__ void wgmma_f16_n128(float (&d)[64], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
                 "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31,"
                 "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47,"
                 "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
                 "%64, %65, p, 1, 1, 0, 0;\n}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
                   "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
                   "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
                   "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
                   "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
                   "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "l"(a), "l"(b), "r"(acc) : "memory");
}
__device__ __forceinline__ void wgmma_s8_n64(uint32_t (&d)[32], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n64k32.s32.s8.s8 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
                 "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
                 "%32, %33, p;\n}\n"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]),
                   "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]),
                   "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]),
                   "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
                 : "l"(a), "l"(b), "r"(acc) : "memory");
}
template <int PREC, int N, class T>
__device__ __forceinline__ void mma(T (&d)[N / 2], uint64_t a, uint64_t b, uint32_t acc) {
    if constexpr (PREC == PREC_TF32 && N == 32) wgmma_tf32_n32(d, a, b, acc);
    else if constexpr (PREC == PREC_TF32 && N == 64) wgmma_tf32_n64(d, a, b, acc);
    else if constexpr (PREC == PREC_BF16 && N == 32) wgmma_bf16_n32(d, a, b, acc);
    else if constexpr (PREC == PREC_BF16 && N == 64) wgmma_bf16_n64(d, a, b, acc);
    else if constexpr (PREC == PREC_BF16 && N == 128) wgmma_bf16_n128(d, a, b, acc);
    else if constexpr (PREC == PREC_F16F && N == 64) wgmma_f16_n64(d, a, b, acc);
    else if constexpr (PREC == PREC_F16F && N == 128) wgmma_f16_n128(d, a, b, acc);
    else if constexpr (PREC == PREC_I8 && N == 64) wgmma_s8_n64(d, a, b, acc);
    else static_assert(N < 0, "no wgmma shape for this precision / query tile");
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from touching accumulator registers across wgmma.wait_group (the tensor core writes them asynchronously)
__device__ __forceinline__ void fence_reg(float& r) { asm volatile("" : "+f"(r)::"memory"); }
__device__ __forceinline__ void fence_reg(uint32_t& r) { asm volatile("" : "+r"(r)::"memory"); }
// an accumulator into the transposition buffer in its own type.  Reading an f32 accumulator as bits (__float_as_uint) makes the compiler
// carry the accumulators through the stage loop as integer values: the copies between the two register types then read accumulators
// between an MMA and its wait, and ptxas serialises the whole wgmma chain (remark C7514; 256-query kernels).
__device__ __forceinline__ void xb_put(uint32_t* d, float x) { *reinterpret_cast<float*>(d) = x; }
__device__ __forceinline__ void xb_put(uint32_t* d, uint32_t x) { *d = x; }

__device__ __forceinline__ uint32_t cluster_ctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// TMA load multicast to the CTAs of `mask`: the box lands at the same shared-memory offset in each, completing on each one's `bar`
__device__ __forceinline__ void tma_load_2d_mc(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar, uint16_t mask) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;"
                 ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(mask) : "memory");
}
// arrive on the barrier at the same offset in CTA `cta` of the cluster
__device__ __forceinline__ void mbar_arrive_cta(uint64_t* bar, uint32_t cta) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(smem_u32(bar)), "r"(cta));
    asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(r) : "memory");
}

__device__ __forceinline__ uint32_t bf16x2_hi(float x, float y, float& rx, float& ry) {
    // hi = bf16_rn(x); the residual x - hi is exact in f32
    __nv_bfloat162 h = __floats2bfloat162_rn(x, y);
    rx = x - __low2float(h); ry = y - __high2float(h);
    return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ uint32_t bf16x2(float x, float y) {
    __nv_bfloat162 h = __floats2bfloat162_rn(x, y);
    return *reinterpret_cast<uint32_t*>(&h);
}

// SCALED (int8 only): 0 = Cosine + ScalarQuantizationI8 (score = the int32 dot product); 1 = Dot + ScalarQuantizationI8 (per-vector
// scale, score = dot_i32 as f32 * query_scale * row_scale, dot_i8_quantized vector_similarity.rs:1754-1758); 2 = Euclidean +
// ScalarQuantizationI8, non-affine (score = -max(0, query_norm + row_norm - 2*dot), euclidean_i8_quantized :1721-1734); 3 = the AFFINE
// variant (integer-valued 0..255 data, euclidean_i8_quantized_affine :1770-1795): the int32 dot product is first corrected for the two zero
// points, dot - zp_row*sum_q(query) - zp_query*sum_q(row) + n*zp_query*zp_row, regrouped as dot - zp_row*sum_q(query) + zp_query*(n*zp_row - sum_q(row))
// Unscaled int8 scores are the int32 dot products as f32 (exact below 2^24), so every variant runs the same f32-score epilogue.
template <int NQ, int PREC, bool BRES, int SCALED, bool PAIR, bool QUEUE>
__global__ void __launch_bounds__(THREADS, 1)
scan_tc(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmA2 /*bf16: lo plane*/,
        const __grid_constant__ CUtensorMap tmBh, const __grid_constant__ CUtensorMap tmBl, uint32_t n_rows, uint32_t n_kchunks, uint32_t n_tiles, uint32_t k,
        const uint32_t* __restrict__ doc_ids, uint64_t* __restrict__ scratch /*[gridDim.y][gridDim.x*4][NQ][32]*/,
        const uint32_t* __restrict__ thr_init /*[gridDim.y*NQ] or null*/, uint32_t nq_valid,
        const uint64_t* __restrict__ ceil_keys /*[gridDim.y*NQ] or null*/, uint32_t nst_rt,
        const uint32_t* __restrict__ del_slot, const uint64_t* __restrict__ del_words /*delete set or null*/,
        const float* __restrict__ row_scale, const float* __restrict__ row_norm /*SCALED: [n_rows]*/,
        const float* __restrict__ q_scale, const float* __restrict__ q_norm /*SCALED: [gridDim.y*NQ]; filter scan: q_scale = margins*/,
        const int2* __restrict__ row_aff /*SCALED 3: [n_rows] (zero_point, dims*zero_point - sum_q)*/, const int2* __restrict__ q_aff /*SCALED 3: [gridDim.y*NQ] (zero_point, sum_q)*/,
        const uint32_t* __restrict__ ivf_sel, uint32_t ivf_words, const uint32_t* __restrict__ row_cluster /*IVF selection mask or null*/,
        uint32_t sample_mode /*write per-(32-row group, query) score maxima instead of lists*/) {
    using C = Cfg<NQ, PREC, BRES, QUEUE>;
    constexpr int TROWS = C::TROWS, MW = C::MW, NQH = C::NQH;
    // 256 queries: the tensor pipe, not HBM, sets the pass time, and the epilogue stalls it -> the common-case test runs on the
    // accumulator fragment, without the shared-memory transposition
    constexpr bool FRAG_VOTE = NQ == 256;
    using AccT = typename std::conditional<PREC == PREC_I8, uint32_t, float>::type;
    const uint32_t STAGES = BRES ? nst_rt : (uint32_t)C::STAGES;
    // the swizzled tiles need 1024-byte alignment in the shared window (the same offset in both CTAs of a pair)
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* base = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t* stage0 = base;
    // QUEUE (256 queries, seeded scan; chosen at launch): chunks with a candidate go through the record queue to the list warps, one
    // list per query per CTA.  Unseeded (no sample pass: delete set, IVF mask, < 65536 rows) the first tiles are an insert storm that the
    // 8 consumer warps clear faster than 3 list warps, so the other instantiation keeps the per-warp lists, inserts in the consumers and
    // gives the producer warpgroup's registers to them, as in the 64/128-query kernels.
    // per-query sorted lists live directly in this CTA's slice of the output scratch (global, L2-resident): they are
    // touched only on the rare candidate insert, and each list is always owned by the same warp
    uint64_t* lists = scratch + ((size_t)blockIdx.y * gridDim.x + blockIdx.x) * (QUEUE ? 1 : 4) * NQ * LIST;   // [QUEUE ? 1 : 4][NQ][32]
    uint8_t* bres = base + STAGES * C::STAGE_BYTES;                           // BRES: resident query block
    uint32_t* xbuf = (uint32_t*)(bres + (BRES ? n_kchunks * C::B_BYTES : 0)); // [8 consumer warps | QSLOTS records][32][XB_STRIDE]
    volatile uint32_t* qstate = xbuf + QSLOTS * REC_WORDS;                    // 256 queries: [QSLOTS] slot states
    volatile uint32_t* qmeta = qstate + QSLOTS;                               //              [QSLOTS][2] (tile, consumer warp 0-3)
    volatile uint32_t* qdone = qmeta + 2 * QSLOTS;                            //              consumer warps finished
    uint32_t* thr_u = xbuf + C::XB_REGION / 4;    // [NQ] ordered-uint score thresholds
    float* qs_sm = (float*)(thr_u + NQ);          // [NQ] SCALED: query scale; filter scan: margin
    float* qn_sm = qs_sm + NQ;                    // [NQ] SCALED: query norm
    uint64_t* bars = (uint64_t*)(thr_u + 3 * NQ);
    uint64_t* full = bars;                     // [STAGES]
    uint64_t* empty = full + MAX_STAGES;       // [STAGES]
    uint64_t* bfull = empty + MAX_STAGES;      // BRES: query block landed

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t group = blockIdx.y;
    const uint32_t rank = PAIR ? cluster_ctarank() : 0u;

    if (threadIdx.x == 0) {
        mbar_init(bfull, 1);
        // every consumer warp releases a stage (and in a pair also the peer's copy of it: the peer's multicast writes into this one)
        for (uint32_t s = 0; s < STAGES; s++) { mbar_init(&full[s], 1); mbar_init(&empty[s], PAIR ? 16 : 8); }
        fence_mbar_init();
    }
    for (int i = threadIdx.x; i < NQ; i += THREADS) {  // seeded by the pre-sample pass when present
        thr_u[i] = blockIdx.y * NQ + i >= nq_valid ? 0xFFFFFFFFu   // zero-padded query slot: unreachable threshold
                                                   : (thr_init ? __ldg(&thr_init[blockIdx.y * NQ + i]) : 0u);
        if (PREC == PREC_F16F) qs_sm[i] = __ldg(&q_scale[blockIdx.y * NQ + i]);   // filter scan: per-query margin 2 eps_q
        if (SCALED) { qs_sm[i] = __ldg(&q_scale[blockIdx.y * NQ + i]); qn_sm[i] = SCALED >= 2 ? __ldg(&q_norm[blockIdx.y * NQ + i]) : 0.f; }
    }
    if (QUEUE && threadIdx.x < QSLOTS) qstate[threadIdx.x] = 0u;
    if (QUEUE && threadIdx.x == 0) *qdone = 0u;
    __syncthreads();
    if (PAIR) cluster_sync_all();                 // both CTAs' barriers are initialised before anything arrives on them

    // a pair walks pairs of neighbouring tiles; both CTAs take the same number of steps (the peer's multicast feeds both)
    const uint32_t tile0 = PAIR ? (blockIdx.x & ~1u) + rank : blockIdx.x;

    // The exact candidate test and list insert for one 8-query chunk c of 32 rows: lane = corpus row `row`, its CHUNK scores (f32 bits)
    // at xr[0..CHUNK).  Per column: ballot of the rows at or above the query's threshold, delete set / IVF mask / paging ceiling, then
    // one insert per key or (warm-up tiles: many rows pass) a bulk sort + merge into the list, and the threshold rises to its k-th
    // best (filter scan: lowered by the query's margin).  A runtime loop keeps one copy of this path.  QUEUE kernels run only seeded,
    // and a delete set or an IVF mask turns the seed off (the launcher checks it): they have no delete / IVF test.
    auto insert_chunk = [&](const uint32_t* xr, uint32_t row, bool valid, int c, uint64_t* qlists) {
#pragma unroll 1
        for (int j = 0; j < CHUNK; j++) {
            const int q = c * CHUNK + j;
            const float sc = __uint_as_float(xr[j]);
            const uint32_t so = ord_f32(sc);
            const bool pass = valid && sc == sc && so >= thr_u[q];
            unsigned pm = __ballot_sync(FULL, pass);
            if (!pm) continue;
            uint64_t key = 0;
            if (pass) {
                const uint32_t doc = doc_ids ? __ldg(&doc_ids[row]) : row;
                key = ((uint64_t)so << 32) | (uint64_t)(0xFFFFFFFFu - (PREC == PREC_F16F ? row : doc));   // filter scan: candidates are named by row
                if (!QUEUE && (doc_deleted(del_slot, del_words, doc) || ivf_skipped(ivf_sel, ivf_words, blockIdx.y * NQ + q, row_cluster, row))) key = 0;
            }
            if (ceil_keys || (!QUEUE && (del_slot || ivf_sel))) {   // paging: keys >= ceil were returned by an earlier page (0 = exhausted)
                if (ceil_keys) { const uint64_t ceil = __ldg(&ceil_keys[blockIdx.y * NQ + q]); if (key >= ceil) key = 0; }
                pm = __ballot_sync(FULL, key != 0);
                if (!pm) continue;
            }
            uint64_t L = qlists[q * LIST + lane];
            if (__popc(pm) > 3) {
                L = wl_merge(L, wl_sort_desc(key, lane), lane);
            } else {
                while (pm) { const int src = __ffs(pm) - 1; pm &= pm - 1; wl_insert(L, shfl64(key, src), lane); }
            }
            qlists[q * LIST + lane] = L;
            uint32_t kth = (uint32_t)(shfl64(L, (int)k - 1) >> 32);
            if (PREC == PREC_F16F && kth) kth = ord_f32(__fsub_rd(unord_f32(kth), qs_sm[q]));   // candidates: s^ >= k-th best s^ - 2 eps_q
            if (lane == 0 && kth > thr_u[q]) atomicMax(&thr_u[q], kth);
        }
    };

    if (warp < 4) {
        // QUEUE: warps 1-3 run the list inserts and need more than the producer's registers
        if constexpr (QUEUE) asm volatile("setmaxnreg.dec.sync.aligned.u32 64;");
        else asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        // ===================== TMA producer =====================
        if (warp == 0 && lane == 0) {
            tma_prefetch_desc(&tmA); tma_prefetch_desc(&tmA2); tma_prefetch_desc(&tmBh); tma_prefetch_desc(&tmBl);
            uint32_t it = 0;
            if (BRES) {
                mbar_arrive_expect_tx(bfull, n_kchunks * C::B_BYTES);
                for (uint32_t kc = 0; kc < n_kchunks; ++kc)
                    tma_load_2d(bres + kc * C::B_BYTES, &tmBh, (int)(kc * C::KCE), (int)(group * NQ), bfull);
            }
            for (uint32_t tile = tile0; tile - rank < n_tiles; tile += gridDim.x) {
                for (uint32_t kc = 0; kc < n_kchunks; ++kc, ++it) {
                    uint32_t s = it % STAGES, ph = (it / STAGES) & 1u;
                    uint8_t* st = stage0 + s * C::STAGE_BYTES;
                    mbar_wait(&empty[s], ph ^ 1u);
                    mbar_arrive_expect_tx(&full[s], C::TX_BYTES);
                    tma_load_2d(st, &tmA, (int)(kc * C::KCE), (int)(tile * TROWS), &full[s]);
                    if (PREC == PREC_BF16) tma_load_2d(st + C::A2_OFF, &tmA2, (int)(kc * C::KCE), (int)(tile * TROWS), &full[s]);   // lo plane
                    if (PAIR)   // this CTA's half of the query block, into both CTAs
                        tma_load_2d_mc(st + C::B_OFF + rank * (C::B_BYTES / 2), &tmBh, (int)(kc * C::KCE), (int)(group * NQ + rank * NQH), &full[s], (uint16_t)3);
                    else if (!BRES)
                        tma_load_2d(st + C::B_OFF, &tmBh, (int)(kc * C::KCE), (int)(group * NQ), &full[s]);
                    if (PREC == PREC_TF32 || PREC == PREC_BF16) tma_load_2d(st + C::B_OFF + C::B_BYTES, &tmBl, (int)(kc * C::KCE), (int)(group * NQ), &full[s]);
                }
            }
        } else if (QUEUE && warp > 0) {
            // ===================== list warps (QUEUE): drain the record queue =====================
            // List warp r owns the 8-query chunks c with c % 3 == r, so every (CTA, query) list has one writer.  It exits once all
            // 8 consumer warps have finished and no record of its chunks is left.
            const uint32_t r = (uint32_t)warp - 1u;
            for (uint32_t c = r; c < NQ / CHUNK; c += 3)
                for (int i = lane; i < CHUNK * LIST; i += 32) lists[c * CHUNK * LIST + i] = 0;
            __syncwarp();
            for (;;) {
                const bool fin = *qdone == 8u;   // read before the states: every record published before the count is seen below
                __threadfence_block();
                const uint32_t f = lane < QSLOTS ? qstate[lane] : 0u;
                unsigned ready = __ballot_sync(FULL, f >= 2u && (f - 2u) % 3u == r);
                if (!ready) {
                    if (fin) break;
                    __nanosleep(128);
                    continue;
                }
                __threadfence_block();
                while (ready) {
                    const int s = __ffs(ready) - 1; ready &= ready - 1;
                    const uint32_t tile = qmeta[2 * s], w = qmeta[2 * s + 1];
                    const int c = (int)__shfl_sync(FULL, f, s) - 2;
                    const uint32_t row = tile * TROWS + (uint32_t)(64 * (lane >> 4) + 16 * w + (lane & 15));
                    insert_chunk(xbuf + s * REC_WORDS + lane * XB_STRIDE, row, row < n_rows, c, lists);
                    __syncwarp();
                    if (lane == 0) { __threadfence_block(); qstate[s] = 0u; }
                }
            }
        }
    } else {
        // the warpgroups trade registers within the CTA's allocation, 384 x 168 = 64512: 128 x 40 + 256 x 232, or with the list warps
        // 128 x 64 + 256 x 216 (an inc beyond what the decs released never returns)
        if constexpr (QUEUE) asm volatile("setmaxnreg.inc.sync.aligned.u32 216;");
        else asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
        // ===================== consumers: MMA + epilogue =====================
        const int cw = (warp - 4) >> 2;          // consumer warpgroup: query columns [cw*NQH, (cw+1)*NQH)
        const int w = warp & 3;                  // rows 16w..16w+15 of every 64-row sub-tile; list w
        const int q0 = cw * NQH;
        uint32_t* xb = xbuf + (warp - 4) * 32 * XB_STRIDE;
        uint64_t* mylists = lists + (size_t)w * NQ * LIST;   // no queue: list w of the warpgroup's queries
        if (!QUEUE && !sample_mode)
            for (int i = lane; i < NQH * LIST; i += 32) mylists[q0 * LIST + i] = 0;
        __syncwarp();
        uint32_t* gmaxu = (uint32_t*)scratch;     // sample mode: ordered-uint group maxima [gridDim.y * NQ][n_tiles * TROWS / 32]
        const uint32_t n_rg = n_tiles * (TROWS / 32);
        AccT acc[MW][NQH / 2];
        if (BRES) mbar_wait(bfull, 0);
        uint32_t it = 0;
        for (uint32_t tile = tile0; tile - rank < n_tiles; tile += gridDim.x) {
            for (uint32_t kc = 0; kc < n_kchunks; ++kc, ++it) {
                const uint32_t s = it % STAGES, ph = (it / STAGES) & 1u;
                uint8_t* st = stage0 + s * C::STAGE_BYTES;
                mbar_wait(&full[s], ph);
                if (PREC == PREC_TF32) {
                    // f32 corpus tile -> (hi in place, lo) operand tiles, by all 256 consumer threads, then visible to the tensor core
                    const int t = threadIdx.x - 128;
                    uint4* A = (uint4*)st;
                    uint4* Al = (uint4*)(st + C::ALO_OFF);
#pragma unroll
                    for (int j = 0; j < (C::A_BYTES / 16) / 256; j++) {
                        uint4 x = A[t + 256 * j], h, l;
                        h.x = x.x & 0xFFFFE000u; h.y = x.y & 0xFFFFE000u; h.z = x.z & 0xFFFFE000u; h.w = x.w & 0xFFFFE000u;
                        l.x = __float_as_uint(__uint_as_float(x.x) - __uint_as_float(h.x));
                        l.y = __float_as_uint(__uint_as_float(x.y) - __uint_as_float(h.y));
                        l.z = __float_as_uint(__uint_as_float(x.z) - __uint_as_float(h.z));
                        l.w = __float_as_uint(__uint_as_float(x.w) - __uint_as_float(h.w));
                        A[t + 256 * j] = h;
                        Al[t + 256 * j] = l;
                    }
                    fence_proxy_async();          // generic-proxy smem writes -> visible to the tensor core (async proxy)
                    asm volatile("bar.sync 1, 256;" ::: "memory");
                }
                const uint32_t sa = smem_u32(st);
                const uint32_t sb = (BRES ? smem_u32(bres + kc * C::B_BYTES) : sa + C::B_OFF) + q0 * C::B_ROW;   // this warpgroup's queries
                wg_fence();
                if (PREC == PREC_I8 || PREC == PREC_F16F) {   // one product; 4 x 32 bytes of K inside the 128-byte swizzle row
                    const uint64_t a = gmma_desc_k128(sa), b = gmma_desc_k128(sb);
#pragma unroll
                    for (int m = 0; m < MW; m++) {
                        const uint64_t am = (uint64_t)((m * 64 * 128) >> 4);
#pragma unroll
                        for (uint32_t kk = 0; kk < 4; kk++)
                            mma<PREC, NQH>(acc[m], a + am + (uint64_t)(kk * 2), b + (uint64_t)(kk * 2), (kc | kk) != 0);
                    }
                } else if (PREC == PREC_TF32) {
                    const uint64_t a_hi = gmma_desc_k128(sa), a_lo = gmma_desc_k128(sa + C::ALO_OFF);
                    const uint64_t b_hi = gmma_desc_k128(sb), b_lo = gmma_desc_k128(sb + C::B_BYTES);
#pragma unroll
                    for (int m = 0; m < MW; m++) {
                        const uint64_t am = (uint64_t)((m * 64 * 128) >> 4);   // next 64-row sub-tile
#pragma unroll
                        for (uint32_t kk = 0; kk < 4; kk++) {        // 4 x K=8 (32 bytes) inside the 128-byte swizzle row
                            const uint64_t o = (uint64_t)(kk * 2);  // +32 bytes in 16-byte units
                            mma<PREC, NQH>(acc[m], a_hi + am + o, b_hi + o, (kc | kk) != 0);
                            mma<PREC, NQH>(acc[m], a_lo + am + o, b_hi + o, 1);
                            mma<PREC, NQH>(acc[m], a_hi + am + o, b_lo + o, 1);
                        }
                    }
                } else {
                    const uint64_t a1 = gmma_desc_k64(sa + C::ALO_OFF), a2 = gmma_desc_k64(sa + C::A2_OFF);
                    const uint64_t b1 = gmma_desc_k64(sb), b2 = gmma_desc_k64(sb + C::B_BYTES);
#pragma unroll
                    for (int m = 0; m < MW; m++) {
                        const uint64_t am = (uint64_t)((m * 64 * 64) >> 4);   // bf16 sub-tile = 4 KB
#pragma unroll
                        for (uint32_t kk = 0; kk < 2; kk++) {        // 2 x K=16 bf16 (32 bytes) inside the 64-byte swizzle row
                            const uint64_t o = (uint64_t)(kk * 2);
                            mma<PREC, NQH>(acc[m], a1 + am + o, b1 + o, (kc | kk) != 0);
                            mma<PREC, NQH>(acc[m], a2 + am + o, b1 + o, 1);
                            mma<PREC, NQH>(acc[m], a1 + am + o, b2 + o, 1);
                        }
                    }
                }
                wg_commit();
                wg_wait<1>();                                  // the previous stage's MMAs retired: release it
                if (kc > 0 && lane == 0) {
                    const uint32_t sp = (it - 1) % STAGES;
                    mbar_arrive(&empty[sp]);
                    if (PAIR) mbar_arrive_cta(&empty[sp], rank ^ 1u);
                }
            }
            wg_wait<0>();
            if (lane == 0) {
                const uint32_t sp = (it - 1) % STAGES;
                mbar_arrive(&empty[sp]);
                if (PAIR) mbar_arrive_cta(&empty[sp], rank ^ 1u);
            }
#pragma unroll
            for (int m = 0; m < MW; m++)
#pragma unroll
                for (int i = 0; i < NQH / 2; i++) fence_reg(acc[m][i]);

            // ===================== epilogue: accumulators -> filter -> per-warp per-query top-k (no CTA-level barriers) =====================
            // The per-query threshold (ordered-uint score of the best k-th entry any warp of the warpgroup has seen, seeded by the
            // pre-sample pass) is shared through smem with atomicMax: monotone, so stale reads only cost an extra insert.
            // Fragment of m64nN: register 4j+2h+b of sub-tile m holds row 16w + lane/4 + 8h, column 8j + 2(lane%4) + b.
#pragma unroll
            for (int p = 0; p < MW / 2; p++) {                        // 32 rows: lanes 0-15 sub-tile 2p, lanes 16-31 sub-tile 2p+1
                const uint32_t row = tile * TROWS + (uint32_t)(64 * (2 * p + (lane >> 4)) + 16 * w + (lane & 15));
                const bool valid = row < n_rows;
                float rs = 0.f, rn = 0.f;
                int2 ra = make_int2(0, 0);
                if (SCALED) {
                    rs = valid ? __ldg(&row_scale[row]) : 0.f;
                    rn = (SCALED >= 2 && valid) ? __ldg(&row_norm[row]) : 0.f;
                    ra = (SCALED == 3 && valid) ? __ldg(&row_aff[row]) : make_int2(0, 0);
                }
#pragma unroll
                for (int jb = 0; jb < NQH / CHUNK; jb++) {
                    const int c = q0 / CHUNK + jb;                    // 8-query chunk of the block
                    if constexpr (FRAG_VOTE && !QUEUE) if (sample_mode) {   // (QUEUE kernels never run the sample pass)
                        // sample pass, in the fragment layout: per column the best of the lane's 4 rows (2 sub-tiles x 2 rows), then
                        // of the 8 lanes that share lane % 4 -> the group maximum over the same 32 rows as the transposed path below
                        // stores, bit for bit (a max of ordered-uint values does not depend on the order it is taken in)
                        uint32_t mx[2] = {0u, 0u};
#pragma unroll
                        for (int hm = 0; hm < 2; hm++)
#pragma unroll
                            for (int h = 0; h < 2; h++)
#pragma unroll
                                for (int b = 0; b < 2; b++) {
                                    const uint32_t r = tile * TROWS + (uint32_t)(64 * (2 * p + hm) + 16 * w + (lane >> 2) + 8 * h);
                                    const float sc = acc[2 * p + hm][4 * jb + 2 * h + b];
                                    uint32_t so = (r < n_rows && sc == sc) ? ord_f32(sc) : 0u;
                                    if (ceil_keys && so) {   // paging: rows already returned by an earlier page do not count
                                        const uint64_t key = ((uint64_t)so << 32) | (uint64_t)(0xFFFFFFFFu - (doc_ids ? __ldg(&doc_ids[r]) : r));
                                        if (key >= __ldg(&ceil_keys[blockIdx.y * NQ + c * CHUNK + 2 * (lane & 3) + b])) so = 0u;
                                    }
                                    mx[b] = max(mx[b], so);
                                }
#pragma unroll
                        for (int m = 4; m < 32; m <<= 1) { mx[0] = max(mx[0], __shfl_xor_sync(FULL, mx[0], m)); mx[1] = max(mx[1], __shfl_xor_sync(FULL, mx[1], m)); }
                        if (lane < 4) {
                            uint32_t* g = gmaxu + (size_t)(blockIdx.y * NQ + c * CHUNK + 2 * lane) * n_rg + (tile * (TROWS / 32) + p * 4 + w);
                            g[0] = mx[0]; g[n_rg] = mx[1];
                        }
                        continue;
                    }
                    if (FRAG_VOTE && !sample_mode) {
                        // common case, in the fragment layout: the lane's 8 scores of the chunk (2 sub-tiles x 2 rows x its 2 columns)
                        // against the thresholds of its 2 columns, one vote.  A superset of the exact per-column test below: float
                        // compare treats -0 = +0 and rejects NaN scores; ord values at or below ord(-inf) (0 = no threshold yet) accept
                        // every score; rows past n_rows are left to the exact test.
                        const uint2 t = *reinterpret_cast<const uint2*>(thr_u + c * CHUNK + 2 * (lane & 3));
                        const float t0 = unord_f32(max(t.x, ORD_NEG_INF)), t1 = unord_f32(max(t.y, ORD_NEG_INF));
                        bool any = false;
#pragma unroll
                        for (int hm = 0; hm < 2; hm++)
#pragma unroll
                            for (int h = 0; h < 2; h++)
                                any |= (acc[2 * p + hm][4 * jb + 2 * h] >= t0) | (acc[2 * p + hm][4 * jb + 2 * h + 1] >= t1);
                        if (!__any_sync(FULL, any)) continue;
                    }
                    if (QUEUE) {
                        // a candidate: the chunk goes to the list warp that owns it as a record in lane = row layout.  Claim a free
                        // slot (wait while the queue is full: the list warps drain it whatever the consumers do), write, publish.
                        int s;
                        for (;;) {
                            unsigned fr = __ballot_sync(FULL, lane < QSLOTS && qstate[lane] == 0u);
                            int got = -1;
                            if (lane == 0)
                                while (fr) {
                                    const int i = __ffs(fr) - 1; fr &= fr - 1;
                                    if (atomicCAS((uint32_t*)&qstate[i], 0u, 1u) == 0u) { got = i; break; }
                                }
                            s = __shfl_sync(FULL, got, 0);
                            if (s >= 0) break;
                            __nanosleep(64);
                        }
                        uint32_t* rec = xbuf + s * REC_WORDS;
#pragma unroll
                        for (int hm = 0; hm < 2; hm++)
#pragma unroll
                            for (int h = 0; h < 2; h++) {
                                uint32_t* d = rec + (hm * 16 + (lane >> 2) + 8 * h) * XB_STRIDE + 2 * (lane & 3);
                                xb_put(&d[0], acc[2 * p + hm][4 * jb + 2 * h]);
                                xb_put(&d[1], acc[2 * p + hm][4 * jb + 2 * h + 1]);
                            }
                        if (lane == 0) { qmeta[2 * s] = tile; qmeta[2 * s + 1] = (uint32_t)w; }
                        __threadfence_block();
                        __syncwarp();
                        if (lane == 0) qstate[s] = 2u + (uint32_t)c;
                        continue;
                    }
                    __syncwarp();
#pragma unroll
                    for (int hm = 0; hm < 2; hm++)
#pragma unroll
                        for (int h = 0; h < 2; h++) {
                            uint32_t* d = xb + (hm * 16 + (lane >> 2) + 8 * h) * XB_STRIDE + 2 * (lane & 3);
                            xb_put(&d[0], acc[2 * p + hm][4 * jb + 2 * h]);
                            xb_put(&d[1], acc[2 * p + hm][4 * jb + 2 * h + 1]);
                        }
                    __syncwarp();
                    uint32_t v[CHUNK];
#pragma unroll
                    for (int j = 0; j < CHUNK; j++) {
                        v[j] = xb[lane * XB_STRIDE + j];
                        if (PREC == PREC_I8 && !SCALED) v[j] = __float_as_uint((float)(int)v[j]);
                        if (SCALED) {
                            // scaled int8: the accumulators are exact int32 dot products; the score is rebuilt with the reference's
                            // operation order so that it is bit-identical to the CPU path, then treated like an f32 score below
                            int di = (int)v[j];
                            if (SCALED == 3) { const int2 qa = __ldg(&q_aff[blockIdx.y * NQ + c * CHUNK + j]); di = di - ra.x * qa.y + qa.x * ra.y; }
                            const float dotf = __fmul_rn(__fmul_rn((float)di, qs_sm[c * CHUNK + j]), rs);
                            const float sc = SCALED >= 2 ? -fmaxf(__fsub_rn(__fadd_rn(qn_sm[c * CHUNK + j], rn), __fmul_rn(2.0f, dotf)), 0.0f) : dotf;
                            v[j] = __float_as_uint(sc);
                        }
                    }
                    if (sample_mode) {
                        // no lists.  Every (tile, pass, warp) is a group of 32 rows; per query the group's best score goes to
                        // gmax[query][group].  The k-th largest group maximum is a valid lower bound of the k-th best score (k groups
                        // each hold a row at least that good) and, for k << #groups, nearly as tight as an exact k-th of the sample.
                        uint32_t keep = 0;
#pragma unroll
                        for (int j = 0; j < CHUNK; j++) {
                            const float sc = __uint_as_float(v[j]);
                            uint32_t so = (valid && sc == sc) ? ord_f32(sc) : 0u;
                            if (ceil_keys && so) {   // paging: rows already returned by an earlier page do not count
                                const uint64_t key = ((uint64_t)so << 32) | (uint64_t)(0xFFFFFFFFu - (doc_ids ? __ldg(&doc_ids[row]) : row));
                                if (key >= __ldg(&ceil_keys[blockIdx.y * NQ + c * CHUNK + j])) so = 0u;
                            }
                            const uint32_t mx = __reduce_max_sync(FULL, so);
                            if (lane == j) keep = mx;
                        }
                        if (lane < CHUNK)
                            gmaxu[(size_t)(blockIdx.y * NQ + c * CHUNK + lane) * n_rg + (tile * (TROWS / 32) + p * 4 + w)] = keep;
                        continue;
                    }
                    if (!FRAG_VOTE) {   // common case, branch-free: one vote per 8-query chunk instead of one per column (a NaN score maps
                        // above every threshold here and is rejected by the per-column test below)
                        const uint4* t4 = reinterpret_cast<const uint4*>(thr_u + c * CHUNK);
                        const uint4 t0 = t4[0], t1 = t4[1];
                        const bool any = (ord_f32(__uint_as_float(v[0])) >= t0.x) | (ord_f32(__uint_as_float(v[1])) >= t0.y) |
                                         (ord_f32(__uint_as_float(v[2])) >= t0.z) | (ord_f32(__uint_as_float(v[3])) >= t0.w) |
                                         (ord_f32(__uint_as_float(v[4])) >= t1.x) | (ord_f32(__uint_as_float(v[5])) >= t1.y) |
                                         (ord_f32(__uint_as_float(v[6])) >= t1.z) | (ord_f32(__uint_as_float(v[7])) >= t1.w);
                        if (!__any_sync(FULL, any && valid)) continue;
                    }
                    // rare after warm-up: per column, from the lane's own row of the buffer
#pragma unroll
                    for (int j = 0; j < CHUNK; j++) xb[lane * XB_STRIDE + j] = v[j];
                    insert_chunk(xb + lane * XB_STRIDE, row, valid, c, mylists);
                }
            }
        }
        if (QUEUE) {   // every record of this warp is published before the list warps can see the count
            __syncwarp();
            if (lane == 0) { __threadfence_block(); atomicAdd((uint32_t*)qdone, 1u); }
        }
    }
    // a pair: the peer may still be multicasting into this CTA's shared memory / arriving on its barriers
    if (PAIR) cluster_sync_all();
}

// [nq_pad][dpad] f32 -> hi / lo parts: tf32 (f32 containers) or bf16
__global__ void split_queries_tf32(const float* __restrict__ q, float* __restrict__ hi, float* __restrict__ lo, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t x = __float_as_uint(q[i]), h = x & 0xFFFFE000u;
    hi[i] = __uint_as_float(h);
    lo[i] = __uint_as_float(x) - __uint_as_float(h);
}
// queries [nq][dims] f32 -> padded, (Cosine:) L2-normalised exactly like prep_queries (vec_scan.cu), split into bf16 hi / lo parts:
// one launch instead of prep_queries + split
__global__ void prep_split_queries_bf16(const float* __restrict__ q, uint32_t nq, uint32_t dims, uint64_t qstride,
                                        __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, uint32_t nq_pad, uint32_t dpad, int normalize,
                                        float* __restrict__ f32_out /*filter scan: padded f32 queries for the refine step, else null*/,
                                        float* __restrict__ margin_out /*filter scan: [nq_pad] 2 eps_q*/, const uint32_t* __restrict__ row_err /*{max|a-h(a)|, max|h(a)|} bits*/) {
    const int lane = threadIdx.x & 31;
    const uint32_t row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= nq_pad) return;
    const bool filter = margin_out != nullptr;             // filter scan: `hi` receives the scaled fp16 query, `lo` is not written
    __nv_bfloat16* oh = hi + (size_t)row * dpad;
    __nv_bfloat16* ol = lo + (size_t)row * dpad;
    __half* o16 = reinterpret_cast<__half*>(oh);
    float* of = f32_out ? f32_out + (size_t)row * dpad : nullptr;
    if (row >= nq) {
        for (uint32_t i = lane; i < dpad; i += 32) { oh[i] = __float2bfloat16_rn(0.f); if (!filter) ol[i] = __float2bfloat16_rn(0.f); if (of) of[i] = 0.f; }
        if (filter && lane == 0) margin_out[row] = 0.f;
        return;
    }
    const float* src = q + (size_t)row * qstride;
    float f = 1.f;
    if (normalize) {
        float s = 0.f;
        for (uint32_t i = lane; i < dims; i += 32) { float v = src[i]; s = fmaf(v, v, s); }
        for (int m = 16; m; m >>= 1) s += __shfl_xor_sync(FULL, s, m);
        f = 1.0f / sqrtf(s);
    }
    if (!filter) {
        for (uint32_t i = lane; i < dpad; i += 32) {
            const float x = i < dims ? src[i] * f : 0.f;
            const __nv_bfloat16 h = __float2bfloat16_rn(x);
            oh[i] = h;
            ol[i] = __float2bfloat16_rn(x - __bfloat162float(h));
            if (of) of[i] = x;
        }
        return;
    }
    // filter scan: scale the query by a power of two so that its largest element lands in [128, 256) (exact; keeps the small elements
    // out of fp16's subnormal range), round to fp16, and bound the error of s^ for this query
    float mx = 0.f;
    for (uint32_t i = lane; i < dims; i += 32) mx = fmaxf(mx, fabsf(src[i] * f));
    for (int m = 16; m; m >>= 1) mx = fmaxf(mx, __shfl_xor_sync(FULL, mx, m));
    const float sb = (mx > 0.f && mx < 3.0e38f) ? exp2f((float)(7 - ilogbf(mx))) : 1.f;
    float nb2 = 0.f, eb2 = 0.f;   // |b|^2 and |b - h(b)|^2 of the scaled query
    for (uint32_t i = lane; i < dpad; i += 32) {
        const float x = i < dims ? src[i] * f : 0.f;
        const float xs = x * sb;
        const __half h = __float2half_rn(xs);
        const float r = xs - __half2float(h);
        o16[i] = h;
        if (of) of[i] = x;
        nb2 = fmaf(xs, xs, nb2); eb2 = fmaf(r, r, eb2);
    }
    // eps_q >= |s - s^| for every row: |a.b - h(a).h(b)| = |(a - h(a)).b + h(a).(b - h(b))| <= E_a |b| + H_a |b - h(b)| (Cauchy-Schwarz, E_a / H_a =
    // the row maxima computed at load time), plus the f32 accumulation slack of the tensor core (truncating adds: <= 2^-23 of the absolute
    // sum per element) and of the refine dot product (<= 2^-24): dpad * 2^-22 * H_a |b| covers both with room.  1.001 absorbs the rounding
    // of this arithmetic itself.
    for (int m = 16; m; m >>= 1) { nb2 += __shfl_xor_sync(FULL, nb2, m); eb2 += __shfl_xor_sync(FULL, eb2, m); }
    if (lane == 0) {
        const float Ea = __uint_as_float(row_err[0]), Ha = __uint_as_float(row_err[1]);
        const float nb = sqrtf(nb2) * 1.00001f, eb = sqrtf(eb2) * 1.00001f;
        const float eps = (Ea * nb + Ha * eb + (float)dpad * 2.38418579e-7f * Ha * nb) * 1.001f;
        margin_out[row] = 2.0f * eps;
    }
}
// load time (filter scan): the fp16 plane h = half_rn(x * scale) (scale = a power of two chosen per index) and the index-wide error bounds
// E_a = max over rows of |x*scale - h|_2, H_a = max over rows of |h|_2, rounded up; one warp per row, maxima kept as f32 bit patterns
// (non-negative floats order like their bits)
__global__ void rows_f16_err(const float* __restrict__ x, __half* __restrict__ h16, uint64_t n, uint32_t dpad, float scale, uint32_t* __restrict__ err) {
    const int lane = threadIdx.x & 31;
    const uint64_t row = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= n) return;
    float e2 = 0.f, h2 = 0.f;
    for (uint32_t i = lane; i < dpad; i += 32) {
        const float xs = x[row * dpad + i] * scale;
        const __half hh = __float2half_rn(xs);
        const float h = __half2float(hh), r = xs - h;
        h16[row * dpad + i] = hh;
        e2 = fmaf(r, r, e2); h2 = fmaf(h, h, h2);
    }
    for (int m = 16; m; m >>= 1) { e2 += __shfl_xor_sync(FULL, e2, m); h2 += __shfl_xor_sync(FULL, h2, m); }
    if (lane == 0) {
        const float e = sqrtf(e2) * 1.00001f, h = sqrtf(h2) * 1.00001f;
        if (!(e < 3.0e38f) || !(h < 3.0e38f)) { atomicMax(&err[0], 0x7F800000u); atomicMax(&err[1], 0x7F800000u); return; }   // NaN / overflowing row: infinite margin -> every query falls back
        atomicMax(&err[0], __float_as_uint(e)); atomicMax(&err[1], __float_as_uint(h));
    }
}
// max |x| over a block of rows (chooses the fp16 scale of a Dot index from its first level); err[0] as f32 bits
__global__ void max_abs_f32(const float* __restrict__ x, size_t n, uint32_t* __restrict__ out) {
    float m = 0.f;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) { const float v = fabsf(x[i]); if (v < 3.0e38f) m = fmaxf(m, v); }
    for (int s = 16; s; s >>= 1) m = fmaxf(m, __shfl_xor_sync(FULL, m, s));
    if ((threadIdx.x & 31) == 0) atomicMax(out, __float_as_uint(m));
}

// load time: (normalised) f32 corpus rows -> the two bf16 planes the tensor-core scan streams (hi = bf16_rn(x), lo = bf16_rn(x - hi))
__global__ void split_rows_bf16(const float* __restrict__ x, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float v = x[i];
    const __nv_bfloat16 h = __float2bfloat16_rn(v);
    hi[i] = h;
    lo[i] = __float2bfloat16_rn(v - __bfloat162float(h));
}

// thr[q] = ordered-uint of the k-th largest of gmax[q][0..n_rg) as an f32 score (0 = no threshold when fewer than k groups
// hold an eligible row).  One warp per query, lane-distributed sorted list, chunks that cannot enter the list are skipped.
__global__ void __launch_bounds__(256)
kth_from_groupmax(const int* __restrict__ gmax, uint32_t n_rg, uint32_t nq, uint32_t k, uint32_t* __restrict__ thr,
                  int is_int /*1: int32 dot products (INT_MIN = none), 0: ordered-uint f32 scores (0 = none)*/,
                  const float* __restrict__ margin /*filter scan: thr = k-th - margin[q]; else null*/) {
    // one CTA per query: 8 warps each reduce a slice of the group maxima to a sorted top-32, warp 0 merges the 8 lists (one warp per
    // query walked n_rg / 32 dependent iterations: 57 us under ncu for 2368 groups x 256 queries, as long as the sample scan itself)
    __shared__ uint64_t sm[8][LIST];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t q = blockIdx.x;
    const int* g = gmax + (size_t)q * n_rg;
    uint64_t L = 0;
    for (uint32_t base = warp * 32; base < n_rg; base += 256) {
        const uint32_t i = base + lane;
        // key: order-preserving unsigned value in the high word (> 0 for every eligible row), group index below it keeps keys distinct
        const uint32_t u = i < n_rg ? ((uint32_t)g[i] ^ (is_int ? 0x80000000u : 0u)) : 0u;
        const uint64_t key = u == 0u ? 0ull : ((uint64_t)u << 32) | (uint64_t)(0xFFFFFFFFu - i);
        const uint64_t kth = shfl64(L, (int)k - 1);
        if (__any_sync(FULL, key > kth)) L = wl_merge(L, wl_sort_desc(key, lane), lane);
    }
    sm[warp][lane] = L;
    __syncthreads();
    if (warp != 0) return;
    for (int w = 1; w < 8; w++) L = wl_merge(L, sm[w][lane], lane);
    const uint64_t kth = shfl64(L, (int)k - 1);
    if (lane == 0) {
        uint32_t t = !kth ? 0u : (is_int ? ord_f32((float)(int)((uint32_t)(kth >> 32) ^ 0x80000000u)) : (uint32_t)(kth >> 32));
        if (t && margin) t = ord_f32(__fsub_rd(unord_f32(t), margin[q]));
        thr[q] = t;
    }
}

}  // namespace tc

template <int NQ, int PREC, bool BRES = false, int SCALED = 0, bool PAIR = false>
static int32_t launch_tc_n(const ScanArgs& a, cudaStream_t st) {
    using C = tc::Cfg<NQ, PREC, BRES>;
    static_assert(!PAIR || (NQ == 256 && PREC == tc::PREC_F16F && !BRES), "CTA pairs run the 256-query filter scan only");
    CUtensorMap tmA, tmA2, tmBh, tmBl;
    uint32_t n_tiles = (uint32_t)((a.n_rows + C::TROWS - 1) / C::TROWS);
    uint32_t n_groups = a.nq_pad / NQ;
    size_t nel = (size_t)a.nq_pad * a.dpad;
    uint32_t n_kchunks = a.dpad / tc::KC;
    if constexpr (PREC == tc::PREC_I8) {
        // int8 corpus / queries (quantised by the caller): 128 dims per 128-byte swizzle row
        SSB_TRY(encode_tmap_2d(&tmA, a.rows_i8, 1, a.dpad8, a.n_rows, a.dpad8, 128, C::TROWS, 128));
        SSB_TRY(encode_tmap_2d(&tmBh, a.queries_i8, 1, a.dpad8, a.nq_pad, a.dpad8, 128, NQ, 128));
        tmBl = tmBh; tmA2 = tmA;
        n_kchunks = a.dpad8 / 128;
    } else if constexpr (PREC == tc::PREC_TF32) {
        SSB_TRY(encode_tmap_2d_f32(&tmA, a.rows, a.dpad, a.n_rows, (uint64_t)a.dpad * 4, tc::KC, C::TROWS, 1));
        SSB_TRY(encode_tmap_2d_f32(&tmBh, a.q_hi, a.dpad, a.nq_pad, (uint64_t)a.dpad * 4, tc::KC, NQ, 1));
        SSB_TRY(encode_tmap_2d_f32(&tmBl, a.q_lo, a.dpad, a.nq_pad, (uint64_t)a.dpad * 4, tc::KC, NQ, 1));
        tmA2 = tmA;
        if (!a.thr_init) tc::split_queries_tf32<<<(unsigned)((nel + 255) / 256), 256, 0, st>>>(a.queries_padded, a.q_hi, a.q_lo, nel);
    } else if constexpr (PREC == tc::PREC_F16F) {
        // filter scan: fp16 plane and fp16 queries only, 64 halves (128 bytes) per swizzle row; the box may run past dpad (zero fill).
        // A pair loads the query block in two halves, one per CTA.
        if (!a.rows_h16 || !a.q_scale) { set_error("tensor-core filter scan: the index holds no fp16 plane / no margins"); return SSB_E_STATE; }
        SSB_TRY(encode_tmap_2d(&tmA, a.rows_h16, 2 /*fp16: 2-byte elements*/, a.dpad, a.n_rows, (uint64_t)a.dpad * 2, 64, C::TROWS, 128));
        SSB_TRY(encode_tmap_2d(&tmBh, a.q_hi, 2, a.dpad, a.nq_pad, (uint64_t)a.dpad * 2, 64, PAIR ? NQ / 2 : NQ, 128));
        tmBl = tmBh; tmA2 = tmA;
        n_kchunks = (a.dpad + 63) / 64;
    } else {
        // corpus: the two bf16 planes written at load time; queries: the two bf16 parts live in the q_hi / q_lo buffers (half of
        // each is used) and were written by prep_split_queries_bf16 (launch_prep_split_queries_bf16)
        if (!a.rows_hi || !a.rows_lo) { set_error("tensor-core bf16 scan: the index holds no bf16 planes"); return SSB_E_STATE; }
        SSB_TRY(encode_tmap_2d(&tmA, a.rows_hi, 2 /*bf16*/, a.dpad, a.n_rows, (uint64_t)a.dpad * 2, tc::KC, C::TROWS, 64));
        SSB_TRY(encode_tmap_2d(&tmA2, a.rows_lo, 2 /*bf16*/, a.dpad, a.n_rows, (uint64_t)a.dpad * 2, tc::KC, C::TROWS, 64));
        SSB_TRY(encode_tmap_2d(&tmBh, a.q_hi, 2 /*bf16*/, a.dpad, a.nq_pad, (uint64_t)a.dpad * 2, tc::KC, NQ, 64));
        SSB_TRY(encode_tmap_2d(&tmBl, a.q_lo, 2 /*bf16*/, a.dpad, a.nq_pad, (uint64_t)a.dpad * 2, tc::KC, NQ, 64));
    }
    // one CTA per SM at most; a pair per two SMs, both CTAs of a pair on the tiles of one pair of neighbouring tiles
    uint32_t gx = n_tiles < (uint32_t)a.n_sms ? n_tiles : (uint32_t)a.n_sms;
    if (PAIR) {
        uint32_t n_pairs = (n_tiles + 1) / 2, n_clusters = (uint32_t)a.n_sms / 2;
        gx = 2 * (n_pairs < n_clusters ? n_pairs : n_clusters);
    }
    // the seeded 256-query scan runs the record-queue instantiation (no delete / IVF test in it: either turns the seed off anyway).
    // Lists per CTA: one per consumer warp of a warpgroup, or with the queue one per query.
    const bool queue = NQ == 256 && a.thr_init && !a.sample_groupmax && !a.del_slot && !a.ivf_sel;
    using CQ = tc::Cfg<NQ, PREC, BRES, NQ == 256>;
    const uint32_t n_lists = queue ? 1u : 4u;
    if ((size_t)n_groups * gx * n_lists * NQ * LIST * 8 > a.scratch_bytes) { set_error("vector scan scratch too small"); return SSB_E_STATE; }
    uint32_t nst = queue ? CQ::STAGES : C::STAGES;
    int smem = queue ? CQ::SMEM : C::SMEM;
    if (BRES) {   // resident query block + as many corpus stages as fit (tc::i8_resident guarantees >= 3)
        const int fixed = (int)n_kchunks * C::B_BYTES + C::FIXED;
        nst = (uint32_t)((tc::SMEM_MAX - fixed) / C::STAGE_BYTES);
        if (nst > (uint32_t)tc::MAX_STAGES) nst = tc::MAX_STAGES;
        smem = fixed + (int)nst * C::STAGE_BYTES;
    }
    auto kern = queue ? tc::scan_tc<NQ, PREC, BRES, SCALED, PAIR, NQ == 256> : tc::scan_tc<NQ, PREC, BRES, SCALED, PAIR, false>;
    // per launch, not once per process: the opt-in applies to the CURRENT device's context only (ssb_config.device allows
    // several indexes on different GPUs in one process); the call is a cheap host-side attribute write
    SSB_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, BRES ? tc::SMEM_MAX : smem));
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(gx, n_groups); cfg.blockDim = dim3(tc::THREADS); cfg.dynamicSmemBytes = (size_t)smem; cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = PAIR ? 2 : 1; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    cfg.attrs = at; cfg.numAttrs = PAIR ? 1 : 0;
    if (a.ev0) cudaEventRecord(a.ev0, st);
    SSB_CUDA_TRY(cudaLaunchKernelEx(&cfg, kern, tmA, tmA2, tmBh, tmBl, (uint32_t)a.n_rows, n_kchunks, n_tiles,
                                    a.k, a.doc_ids, a.scratch, a.thr_init, a.nq_valid ? a.nq_valid : a.nq_pad, a.ceil_keys, nst,
                                    a.del_slot, a.del_words, a.row_scale, a.row_norm, a.q_scale, a.q_norm,
                                    (const int2*)a.row_aff, (const int2*)a.q_aff,
                                    a.ivf_sel, a.ivf_words, a.row_cluster,
                                    a.sample_groupmax ? 1u : 0u));
    if (a.ev1) cudaEventRecord(a.ev1, st);
    if (a.sample_groupmax) {   // threshold seeding pass: scratch holds gmax[nq_pad][n_tiles * TROWS / 32]
        tc::kth_from_groupmax<<<a.nq_pad, 256, 0, st>>>((const int*)a.scratch, n_tiles * (C::TROWS / 32), a.nq_pad, a.k, a.thr_buf,
                                                        0, PREC == tc::PREC_F16F ? a.q_scale : nullptr);
        SSB_CUDA_TRY(cudaGetLastError());
        if (a.launches) *a.launches += PREC == tc::PREC_TF32 ? 3 : 2;   // (tf32 query split +) scan + kth
        return SSB_OK;
    }
    if (PREC == tc::PREC_F16F && queue && a.unmerged_lists) {   // refine_candidates merges the per-CTA lists of its query itself
        *a.unmerged_lists = gx;
        if (a.launches) *a.launches += 1;   // scan
        return SSB_OK;
    }
    // scratch layout [group][list][q in NQ][32] -> generic merge with qt = NQ
    merge_lists_generic(a.scratch, gx * n_lists, NQ, a.nq_pad, a.keys_out, st);
    SSB_CUDA_TRY(cudaGetLastError());
    if (a.launches) *a.launches += 2;   // scan + merge (the tf32 query split is counted with the sample pass)
    return SSB_OK;
}

static int32_t launch_scan_tc_impl(const ScanArgs& a, Scan s, cudaStream_t st) {
    if (a.n_rows == 0 || a.nq_pad == 0) return SSB_OK;
    if (a.nq_pad % queries_per_pass(s) != 0) { set_error("tensor-core scan: query count must be padded to the %u-query tile", queries_per_pass(s)); return SSB_E_INVALID; }
    if (s != Scan::I8_128 && a.similarity == SSB_SIM_EUCLIDEAN) { set_error("tensor-core scan supports Dot/Cosine only"); return SSB_E_UNSUPPORTED; }
    switch (s) {
    case Scan::Tf32_64: return launch_tc_n<64, tc::PREC_TF32>(a, st);
    case Scan::Tf32_128: return launch_tc_n<128, tc::PREC_TF32>(a, st);
    case Scan::Bf16_64: return launch_tc_n<64, tc::PREC_BF16>(a, st);
    case Scan::Bf16_128: return launch_tc_n<128, tc::PREC_BF16>(a, st);
    case Scan::Bf16_256: return launch_tc_n<256, tc::PREC_BF16>(a, st);
    case Scan::F16f_128: return launch_tc_n<128, tc::PREC_F16F>(a, st);
    case Scan::F16f_256: return launch_tc_n<256, tc::PREC_F16F>(a, st);
    case Scan::F16f_256Pair:   // the seeding pass stays on one CTA per SM
        return a.sample_groupmax ? launch_tc_n<256, tc::PREC_F16F>(a, st) : launch_tc_n<256, tc::PREC_F16F, false, 0, true>(a, st);
    case Scan::I8_128: {
        if (!a.rows_i8 || !a.queries_i8 || a.dpad8 % 128) { set_error("int8 scan: bad arguments"); return SSB_E_INVALID; }
        const bool res = tc::i8_resident(a.dpad8);   // query block resident in smem when it leaves room for >= 3 corpus stages, else streamed per stage
        if (a.i8_scaled) {
            if (!a.row_scale || !a.q_scale || (a.i8_scaled >= 2 && (!a.row_norm || !a.q_norm)) || (a.i8_scaled == 3 && (!a.row_aff || !a.q_aff))) { set_error("scaled int8 scan: missing scale / norm arrays"); return SSB_E_INVALID; }
            if (a.i8_scaled == 3) return res ? launch_tc_n<128, tc::PREC_I8, true, 3>(a, st) : launch_tc_n<128, tc::PREC_I8, false, 3>(a, st);
            if (a.i8_scaled == 1) return res ? launch_tc_n<128, tc::PREC_I8, true, 1>(a, st) : launch_tc_n<128, tc::PREC_I8, false, 1>(a, st);
            return res ? launch_tc_n<128, tc::PREC_I8, true, 2>(a, st) : launch_tc_n<128, tc::PREC_I8, false, 2>(a, st);
        }
        return res ? launch_tc_n<128, tc::PREC_I8, true>(a, st) : launch_tc_n<128, tc::PREC_I8, false>(a, st);
    }
    case Scan::Ffma: break;
    }
    set_error("tensor-core scan: the FP32 scan is launch_scan_ffma"); return SSB_E_INVALID;
}

int32_t launch_scan_tc(const ScanArgs& a, Scan s, cudaStream_t st) {
    // The sample pass writes per-(32-row group, query) score maxima instead of lists (no insert storm) and costs the same for one
    // 256-row tile per CTA as for a handful of tiles: sample one tile per SM.  (An earlier version ran the normal list epilogue
    // over N/128 rows: ~90 us per pass, and ncu showed the full scan's epilogue warps waiting on list loads for candidates that
    // a better seed rejects.)
    const uint64_t trows = queries_per_pass(s) == 256 ? 128 : tc::TROWS;   // rows per stage of the variant that will run
    // sample tiles per SM: the seed is the k-th best of S sampled rows, the full scan then sees ~k*N/S candidates per query, each a
    // ~1 us latency-bound list insert (256 queries: for a list warp, beside the MMAs).  The filter scan streams a pass in half the time of the 3-product scan, so the
    // same insert load weighs twice as much: it samples more (SSB_TC_SAMPLE_TILES overrides; measured in DESIGN.md §3.2c)
    static const int env_tiles = [] { const char* e = getenv("SSB_TC_SAMPLE_TILES"); return e ? atoi(e) : 0; }();
    const int sample_tiles = env_tiles > 0 ? (env_tiles > 16 ? 16 : env_tiles) : ((s == Scan::F16f_256 || s == Scan::F16f_256Pair) ? 2 : 1);
    uint64_t rows = (uint64_t)a.n_sms * trows * sample_tiles;
    if (rows > a.n_rows / 4) rows = a.n_rows / 4 / trows * trows;
    return with_threshold_seed(a, rows, [s, st](const ScanArgs& x) { return launch_scan_tc_impl(x, s, st); });
}

void launch_kth_from_groupmax(const void* gmax, uint32_t n_groups, uint32_t nq, uint32_t k, uint32_t* thr, int is_int, cudaStream_t st) {
    if (nq) tc::kth_from_groupmax<<<nq, 256, 0, st>>>((const int*)gmax, n_groups, nq, k, thr, is_int, nullptr);
}

int32_t launch_prep_split_queries_bf16(const float* q, uint32_t nq, uint32_t dims, uint64_t qstride, void* hi, void* lo, uint32_t nq_pad,
                                       uint32_t dpad, int normalize, cudaStream_t st, float* f32_out, float* margin_out, const uint32_t* row_err) {
    if (nq_pad == 0) return SSB_OK;
    tc::prep_split_queries_bf16<<<(nq_pad + 7) / 8, 256, 0, st>>>(q, nq, dims, qstride, (__nv_bfloat16*)hi, (__nv_bfloat16*)lo, nq_pad, dpad, normalize,
                                                                  f32_out, margin_out, row_err);
    SSB_CUDA_TRY(cudaGetLastError());
    return SSB_OK;
}

int32_t launch_split_rows_bf16(const float* rows, void* hi, void* lo, size_t n_elems, cudaStream_t st) {
    if (n_elems == 0) return SSB_OK;
    tc::split_rows_bf16<<<(unsigned)((n_elems + 255) / 256), 256, 0, st>>>(rows, (__nv_bfloat16*)hi, (__nv_bfloat16*)lo, n_elems);
    SSB_CUDA_TRY(cudaGetLastError());
    return SSB_OK;
}

int32_t launch_rows_f16_err(const float* rows, void* h16, uint64_t n, uint32_t dpad, float scale, uint32_t* err, cudaStream_t st) {
    if (n == 0) return SSB_OK;
    tc::rows_f16_err<<<(unsigned)((n + 7) / 8), 256, 0, st>>>(rows, (__half*)h16, n, dpad, scale, err);
    SSB_CUDA_TRY(cudaGetLastError());
    return SSB_OK;
}
int32_t launch_max_abs_f32(const float* x, size_t n, uint32_t* out_bits, cudaStream_t st) {
    if (n == 0) return SSB_OK;
    tc::max_abs_f32<<<296, 256, 0, st>>>(x, n, out_bits);
    SSB_CUDA_TRY(cudaGetLastError());
    return SSB_OK;
}

size_t scan_tc_scratch_bytes(int n_sms, uint32_t nq_pad) { return (size_t)nq_pad * (size_t)n_sms * 4 * LIST * 8; }

}  // namespace vec
}  // namespace ssb
