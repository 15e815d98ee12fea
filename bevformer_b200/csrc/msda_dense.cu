// Sampler backward: grad_value of the COARSE pyramid levels as a dense product on the tensor cores.
//
//   grad_value[b, pixel, m, :] = sum over the samples that touch `pixel` of  (attn * bilinear weight) * grad_out[row, m, :]
//
// (the col2im half of mmcv's ms_deform_attn_backward; call site
// projects/mmdet3d_plugin/bevformer/modules/multi_scale_deformable_attn_function.py:150-160, arithmetic
// SURVEY.md Appendix A).  The one-kernel backward (msda.cu) issues one 128 B L2 reduction per (sample, corner),
// 45.6 M of them per SpatialCrossAttention launch at base, and L2's reduction-sector rate bounds that kernel.
// On the coarse levels a pixel receives hundreds of contributions, so for one (camera, head) the scatter is a
// sparse matrix  C[pixel, row]  (<= 4 P non-zeros per column and level) times the dense  grad_out[row, 32]  --
// and with <= 512 pixels per bin it is cheap to treat C as DENSE:
//
//   * a CTA owns (value map b, head m, pixel bin, chunk of rows) and keeps  D[bin pixels, 32 channels]  in the
//     registers of two issuer warpgroups (kTiles accumulator tiles of 128 pixels x 32 fp32 channels; warpgroup
//     i holds the tiles t with t % 2 == i, each as two wgmma m64n32 accumulators);
//   * per step of 16 rows, ONE THREAD per (row, level) writes that row's coefficients into a bf16
//     16 x (bin pixels) slab of shared memory in the wgmma "MN-major, SWIZZLE_128B" layout (thread-level
//     16-bit read-modify-writes: a column belongs to one thread, so no atomics), the 16 grad_out rows go
//     into a K-major tile, and the issuer warpgroups run  wgmma.mma_async (M = 64, N = 32, K = 16)  for every
//     64-pixel half of every accumulator tile the step touched;
//   * slabs are multi-buffered (the scatter of step i+1 runs under the MMAs of step i; the issuers release a slab
//     through an mbarrier once wgmma.wait_group has retired its MMAs) and are cleaned by re-zeroing exactly the
//     entries that were written;
//   * at the end of the unit the touched tiles go from the registers through a shared-memory transpose to
//     grad_value as full-line 16 B vector reductions (all-zero pieces are skipped).
//
// Per sample this costs a few THREAD-level instructions instead of four warp-wide reductions; the L2
// reduction traffic of these levels drops from 16 sectors per sample to one flush per (unit, touched pixel).
// Coefficients are rounded to bf16 (relative 2^-9, independent per term); accumulation is fp32.
// Levels too large for this treatment (pixels > the launcher's limit) stay on msda_bwd_d32's reduction path
// (its red_skip mask excludes the levels handled here); grad_loc / grad_attn always come from that kernel.
#include <cuda.h>

#include <cstdlib>
#include <cstring>
#include <mutex>

#include "msda_common.cuh"

namespace bevf {

constexpr int kDnK = 16;                 // sampler rows (reduction index) per step == one MMA K
constexpr int kDnMaxBins = 32;
constexpr int kDnBinLevels = 4;          // levels that may share one bin == scatter thread groups
constexpr int kDnTileBytes = 128 * kDnK * 2;           // one accumulator tile's slab: 128 pixels x 16 rows bf16
constexpr int kDnTransposeBytes = 16 * 144;            // per issuer warp: 16 rows x (32 + 4 pad) floats

struct DenseBins {
    int nbins, L;
    int s0[kDnMaxBins], n[kDnMaxBins];                  // first pixel (flattened over the pyramid), pixel count
    int nlev[kDnMaxBins];
    int lev[kDnMaxBins][kDnBinLevels];                  // levels that intersect the bin
    HostLevels hl;                                      // the host's view of the pyramid (checked on the device)
};

// ---- PTX wrappers (the same instructions gemm.cu uses) -------------------------------------------
namespace dn {
__device__ __forceinline__ uint32_t s32(const void *p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(s32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(s32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    const uint32_t addr = s32(bar);
    uint32_t done = 0;
    do {
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
            "selp.u32 %0, 1, 0, p;\n"
            "}\n"
            : "=r"(done) : "r"(addr), "r"(parity) : "memory");
    } while (!done);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// generic-proxy shared-memory writes -> visible to the tensor core's (async proxy) operand reads
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// wgmma shared-memory descriptor, SWIZZLE_128B (layout type 1 in bits [62,64)).
// A operand (the coefficient slab): MN-major.  64 consecutive pixels (128 B) per reduction row, 8-row groups
// 1024 B apart (SBO), the next 64-pixel chunk 16 rows x 128 B = 2048 B further (LBO).
// B operand (grad_out^T: 32 channel rows x 16 reduction columns): K-major, 8-row groups 1024 B apart.
__device__ __forceinline__ uint64_t desc_sw128(uint32_t addr, uint32_t lbo_bytes) {
    uint64_t d = 0;
    d |= static_cast<uint64_t>((addr & 0x3FFFFu) >> 4);
    d |= static_cast<uint64_t>(lbo_bytes >> 4) << 16;
    d |= static_cast<uint64_t>(1024 >> 4) << 32;
    d |= static_cast<uint64_t>(1) << 62;
    return d;
}
// D[64 pixels x 32 channels] += A (MN-major) . B (K-major), fp32 accumulators in registers
// (warp w of the warpgroup, lane l: d[4 j + 2 h + e] = D[16 w + 8 h + l / 4][8 j + 2 (l % 4) + e])
__device__ __forceinline__ void wgmma_m64n32_amn(float (&d)[16], uint64_t da, uint64_t db) {
    asm volatile("wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, 1, 1, 1, 1, 0;\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                 : "l"(da), "l"(db));
}
template <int N> __device__ __forceinline__ void fence_regs(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// byte offset of coefficient (pixel row `row` of the bin, reduction column k) inside a slab
__device__ __forceinline__ uint32_t slab_off(int row, int k) {
    return ((uint32_t)(row >> 6) << 11) + ((uint32_t)k << 7) + ((((uint32_t)(row >> 3) & 7u) ^ ((uint32_t)k & 7u)) << 4) +
           (((uint32_t)row & 7u) << 1);
}
// volatile global loads: they keep their place among the other volatile instructions (barrier waits, shared-memory
// accesses), i.e. the prefetch of the next step really is issued before this step's work
__device__ __forceinline__ float2 ldg_f2(const float2 *p) {
    float2 v;
    asm volatile("ld.global.nc.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "l"(p));
    return v;
}
__device__ __forceinline__ float ldg_f1(const float *p) {
    float v;
    asm volatile("ld.global.nc.f32 %0, [%1];" : "=f"(v) : "l"(p));
    return v;
}
__device__ __forceinline__ uint4 ldg_u4(const uint4 *p) {
    uint4 v;
    asm volatile("ld.global.nc.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}
__device__ __forceinline__ unsigned short lds16(uint32_t addr) {
    unsigned short h;
    asm volatile("ld.shared.u16 %0, [%1];" : "=h"(h) : "r"(addr) : "memory");
    return h;
}
__device__ __forceinline__ void sts16(uint32_t addr, unsigned short h) {
    asm volatile("st.shared.u16 [%0], %1;" ::"r"(addr), "h"(h) : "memory");
}
__device__ __forceinline__ unsigned short bf16_add(unsigned short old, float x) {
    const float v = __uint_as_float((uint32_t)old << 16) + x;
    return __bfloat16_as_ushort(__float2bfloat16_rn(v));
}
}  // namespace dn

// Thread organisation.  NT scatter teams of 128 threads (team t owns slab t and handles steps t, t + NT, ... of the
// unit) and two issuer warpgroups (even / odd accumulator tiles).  Inside a team ONE THREAD PER SAMPLE: a warp covers
// 32 / P reduction columns x the P points of one level, so every point of a (row, level) sits in the same warp.
// The four corners are written in four rounds; inside a round, lanes that address the same coefficient (two points
// of one row in the same pixel) are found with match.any, the lowest lane adds the summed value with one 16-bit
// read-modify-write -- a column never leaves its warp, so there are no atomics and no cross-warp conflicts.
// Hand-over per step:
//   team:    wait empty[t] -> zero what its leaders wrote in the previous use -> scatter -> grad_out tile ->
//            fence.proxy.async -> arrive full[t]
//   issuers: wait full[t] -> wgmma for every touched 64-pixel half of their tiles -> wgmma.wait_group -> empty[t]
// so the scatter of up to NT - 1 further steps runs under the MMAs of the previous ones.
// grad_value is (NB, gv_S, M, 32) and holds the pixels [gv_base, gv_base + gv_S) of every map: the whole pyramid
// (gv_S = S, gv_base = 0), or the fp32 side buffer of the mixed accumulation (gv_base = its first pixel).
// loc / attn hold the levels [loc_level0, L) of every row: (rows, M, L - loc_level0, P[, 2]) -- the whole pyramid, or
// only the coarse samples the fused SCA forward stores (ScaFuse::coarse_loc, msda_common.cuh)
template <int kTiles, int P, int NT>
__global__ void __launch_bounds__(128 * NT + 256, 1)
msda_bwd_dense_tc(const __grid_constant__ DenseBins bins, const int64_t *__restrict__ level_hw,
                  const int64_t *__restrict__ level_start, const float *__restrict__ loc,
                  const float *__restrict__ attn, const bf16 *__restrict__ grad_out,
                  float *__restrict__ grad_value, const int *__restrict__ map_range, int NB, int gv_S, int gv_base,
                  int M, int L, int chunk_rows, int dbg, int loc_level0) {
    static_assert(P == 4 || P == 8, "points per level: 4 or 8");
    static_assert(kTiles == 4, "accumulator tiles per bin: 2 per issuer warpgroup");
    static_assert(NT >= 1 && NT <= 3, "scatter teams");
    constexpr int kThreadsAll = 128 * NT + 256;
    constexpr int kSlabBytes = kTiles * kDnTileBytes;
    constexpr int kMine = kTiles / 2;                        // accumulator tiles per issuer warpgroup
    constexpr int kColsPerWarp = 32 / P;                     // 4 (P = 8) or 8 (P = 4)
    constexpr int kWarpsPerLevel = kDnK / kColsPerWarp;      // 4 or 2
    constexpr int kLevelsPerPass = 4 / kWarpsPerLevel;       // levels the 4 warps of a team cover at once: 1 or 2
    constexpr int kMaxPass = kDnBinLevels / kLevelsPerPass;  // 4 or 2
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t *slab = smem;                                   // NT x kSlabBytes
    uint8_t *gtile = smem + NT * kSlabBytes;                // NT x 4096 (32 channel rows x 128 B)
    float *tr = reinterpret_cast<float *>(gtile + NT * 4096);                       // 8 issuer warps x 16 x 36 floats
    uint64_t *bar_full = reinterpret_cast<uint64_t *>(reinterpret_cast<uint8_t *>(tr) + 8 * kDnTransposeBytes);
    uint64_t *bar_empty = bar_full + NT;
    uint32_t *s_dirty = reinterpret_cast<uint32_t *>(bar_empty + NT);   // [2 t + use parity]: tiles touched by the step in slab t
    __shared__ int s_h[kMaxLevels], s_w[kMaxLevels], s_start[kMaxLevels];
    __shared__ int s_bad;

    const int tid = threadIdx.x, lane = tid & 31;
    const int team = tid >> 7, tt = tid & 127, tw = tt >> 5;      // teams NT, NT + 1 = the two issuer warpgroups
    const bool is_team = team < NT;

    // ---- set-up: pyramid table (device copy, checked against the host's), barriers, clean slabs
    if (tid == 0) s_bad = 0;
    __syncthreads();
    if (tid < L) {
        s_h[tid] = (int)level_hw[2 * tid];
        s_w[tid] = (int)level_hw[2 * tid + 1];
        s_start[tid] = (int)level_start[tid];
    }
    if (tid == 64 && !host_levels_match(bins.hl, level_hw, level_start, L)) s_bad = 1;
    if (tid == 32) {
        for (int i = 0; i < NT; ++i) { dn::mbar_init(&bar_full[i], 128); dn::mbar_init(&bar_empty[i], 8); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        for (int i = 0; i < 2 * NT; ++i) s_dirty[i] = 0;
    }
    {
        uint4 *z = reinterpret_cast<uint4 *>(smem);
        const int n16 = (NT * kSlabBytes + NT * 4096) / 16;
        for (int i = tid; i < n16; i += kThreadsAll) z[i] = make_uint4(0, 0, 0, 0);
    }
    __syncthreads();
    // spatial_shapes on the device differ from the shapes the launcher planned with: msda_bwd_d32 evaluates the
    // same predicate and then keeps every level on its reduction path
    if (s_bad) return;
    dn::fence_async_smem();
    __syncthreads();

    // ---- unit list: (map, chunk, head, bin), bin fastest
    const int per_chunk = M * bins.nbins;
    int total = 0;
    for (int b = 0; b < NB; ++b) {
        const int n = __ldg(map_range + 2 * b + 1) - __ldg(map_range + 2 * b);
        total += ((n + chunk_rows - 1) / chunk_rows) * per_chunk;
    }

    // scatter role of a team thread: reduction column k, point p; level slot of pass q = q * kLevelsPerPass + lsub
    const int k = (tw % kWarpsPerLevel) * kColsPerWarp + lane / P, pt = lane % P, lsub = tw / kWarpsPerLevel;
    const uint32_t my_slab = dn::s32(slab + (is_team ? team : 0) * kSlabBytes) + ((uint32_t)k << 7);   // + column term
    const uint32_t kx = (uint32_t)k & 7u;
    const uint32_t my_gt = dn::s32(gtile + (is_team ? team : 0) * 4096);
    const bool g_role = is_team && tt < 64;                  // grad_out role: row gk, 8-channel group gc
    const int gk = tt & 15, gc = (tt >> 4) & 3;
    uint32_t nuse = 0;                                       // team: uses of its slab so far (CTA lifetime)
    uint32_t nfull[NT];                                      // issuers: completed waits per slab
#pragma unroll
    for (int i = 0; i < NT; ++i) nfull[i] = 0;
    float acc[kMine][2][16];                                 // issuers: tile 2 i + iw, 64-pixel half h
    // the two CTA-wide meeting points of a unit, reached from the team and the issuer branches
    auto unit_bar = [] { asm volatile("bar.sync 1, %0;" ::"n"(kThreadsAll) : "memory"); };

    // byte offset of pixel row `row` in this thread's column (without the slab base)
    auto row_off = [&](int row) -> uint32_t {
        return ((uint32_t)(row >> 6) << 11) + ((((uint32_t)(row >> 3) & 7u) ^ kx) << 4) + (((uint32_t)row & 7u) << 1);
    };

    for (int u = blockIdx.x; u < total; u += gridDim.x) {
        // ---- decode
        int b = 0, rem = u, ps = 0, pe = 0;
        for (; b < NB; ++b) {
            ps = __ldg(map_range + 2 * b); pe = __ldg(map_range + 2 * b + 1);
            const int cnt = ((pe - ps + chunk_rows - 1) / chunk_rows) * per_chunk;
            if (rem < cnt) break;
            rem -= cnt;
        }
        const int chunk = rem / per_chunk, rem2 = rem - chunk * per_chunk;
        const int m = rem2 / bins.nbins, bin = rem2 - m * bins.nbins;
        const int r_begin = ps + chunk * chunk_rows, r_end = min(pe, r_begin + chunk_rows);
        const int nsteps = (r_end - r_begin + kDnK - 1) / kDnK;
        const int s0 = bins.s0[bin], nb = bins.n[bin];

        if (is_team) {
            // ================================ scatter teams ================================
            const int nlev = bins.nlev[bin];
            int lv[kMaxPass], Hq[kMaxPass], Wq[kMaxPass], lb[kMaxPass];
            bool on[kMaxPass];
            // rec[q]: (byte offset / 2) | 0x8000 of the entries this lane wrote (as the leader of its match set)
            uint32_t rec_a[kMaxPass], rec_b[kMaxPass];
#pragma unroll
            for (int q = 0; q < kMaxPass; ++q) {
                const int slot = q * kLevelsPerPass + lsub;
                on[q] = slot < nlev;
                lv[q] = on[q] ? bins.lev[bin][slot] : 0;
                Hq[q] = s_h[lv[q]]; Wq[q] = s_w[lv[q]]; lb[q] = s_start[lv[q]] - s0;
                rec_a[q] = rec_b[q] = 0;
            }
            struct Smp { float x, y, a; };
            auto load_samples = [&](int step, Smp (&q)[kMaxPass]) {
                const int r = r_begin + step * kDnK + k;
                const bool live = step < nsteps && r < r_end;
#pragma unroll
                for (int i = 0; i < kMaxPass; ++i) {
                    q[i].x = q[i].y = q[i].a = 0.f;
                    if (live && on[i]) {
                        const long long e = (((long long)r * M + m) * (L - loc_level0) + lv[i] - loc_level0) * P + pt;
                        const float2 xy = dn::ldg_f2(reinterpret_cast<const float2 *>(loc) + e);
                        q[i].x = xy.x; q[i].y = xy.y; q[i].a = dn::ldg_f1(attn + e);
                    }
                }
            };
            auto load_gout = [&](int step) -> uint4 {
                const int r = r_begin + step * kDnK + gk;
                if (g_role && step < nsteps && r < r_end)
                    return dn::ldg_u4(reinterpret_cast<const uint4 *>(grad_out + ((long long)r * M + m) * 32 + gc * 8));
                return make_uint4(0, 0, 0, 0);
            };
            auto unscatter = [&]() {
#pragma unroll
                for (int q = 0; q < kMaxPass; ++q) {
                    const uint32_t ra = rec_a[q], rb = rec_b[q];
                    if ((ra | rb) != 0) {
                        if (ra & 0x8000u) dn::sts16(my_slab + ((ra & 0x7fffu) << 1), 0);
                        if (ra & 0x80000000u) dn::sts16(my_slab + (((ra >> 16) & 0x7fffu) << 1), 0);
                        if (rb & 0x8000u) dn::sts16(my_slab + ((rb & 0x7fffu) << 1), 0);
                        if (rb & 0x80000000u) dn::sts16(my_slab + (((rb >> 16) & 0x7fffu) << 1), 0);
                        rec_a[q] = rec_b[q] = 0;
                    }
                }
            };
            // one corner of every lane's sample: lanes with the same target are merged, the lowest one writes
            auto corner_round = [&](bool act, uint32_t off, float cf, int row, uint32_t &dirty) -> uint32_t {
                const uint32_t key = act ? (my_slab + off) : (0xffffff00u | (uint32_t)lane);
                const unsigned peers = __match_any_sync(0xffffffffu, key);
                float sum = cf;
                if (__any_sync(0xffffffffu, (peers & (peers - 1u)) != 0u)) {       // some set has more than one lane
                    sum = 0.f;
                    unsigned rem_set = peers;
                    while (__any_sync(0xffffffffu, rem_set != 0u)) {
                        const int src = rem_set ? (__ffs(rem_set) - 1) : lane;
                        const float t = __shfl_sync(0xffffffffu, cf, src);
                        if (rem_set) { sum += t; rem_set &= rem_set - 1u; }
                    }
                }
                if (act && lane == __ffs(peers) - 1) {
                    dn::sts16(key, dn::bf16_add(dn::lds16(key), sum));
                    dirty |= 1u << (row >> 7);
                    return (off >> 1) | 0x8000u;
                }
                return 0u;
            };
            auto scatter = [&](const Smp (&q)[kMaxPass]) -> uint32_t {
                uint32_t dirty = 0;
#pragma unroll
                for (int i = 0; i < kMaxPass; ++i) {
                    if (i * kLevelsPerPass >= nlev) break;            // team-uniform
                    const int H = Hq[i], W = Wq[i], lbase = lb[i];
                    bool p00 = false, p01 = false, p10 = false, p11 = false;
                    int r00 = 0, r01 = 0, r10 = 0, r11 = 0;
                    float c00 = 0.f, c01 = 0.f, c10 = 0.f, c11 = 0.f;
                    bool maybe = on[i] && q[i].a != 0.f;
                    if (maybe) {
                        // cheap rejection first: a level cut into several bins is scanned once per bin, and most of
                        // its samples fall into another one (same rounding as make_corner: unfused multiply / add)
                        const float yy = __fadd_rn(__fmul_rn(q[i].y, (float)H), -0.5f);
                        maybe = (yy > -1.f) && (yy < (float)H);
                        if (maybe) {
                            const int y0 = (int)floorf(yy);
                            maybe = lbase + (min(y0 + 1, H - 1) + 1) * W > 0 && lbase + max(y0, 0) * W < nb;
                        }
                    }
                    if (__any_sync(0xffffffffu, maybe)) {              // warp-uniform
                        if (maybe) {
                            const Corner c = make_corner(q[i].x, q[i].y, H, W);
                            if (c.valid) {
                                const float a = q[i].a;
                                r00 = lbase + c.pidx; r01 = r00 + c.dx; r10 = r00 + c.dy * W; r11 = r10 + c.dx;
                                c00 = c.w00 * a; c01 = c.w01 * a; c10 = c.w10 * a; c11 = c.w11 * a;
                                p00 = c00 != 0.f && (unsigned)r00 < (unsigned)nb; p01 = c01 != 0.f && (unsigned)r01 < (unsigned)nb;
                                p10 = c10 != 0.f && (unsigned)r10 < (unsigned)nb; p11 = c11 != 0.f && (unsigned)r11 < (unsigned)nb;
                            }
                        }
                        uint32_t ra = 0, rb = 0;
                        ra |= corner_round(p00, p00 ? row_off(r00) : 0u, c00, r00, dirty);
                        ra |= corner_round(p01, p01 ? row_off(r01) : 0u, c01, r01, dirty) << 16;
                        rb |= corner_round(p10, p10 ? row_off(r10) : 0u, c10, r10, dirty);
                        rb |= corner_round(p11, p11 ? row_off(r11) : 0u, c11, r11, dirty) << 16;
                        rec_a[i] = ra; rec_b[i] = rb;
                    }
                }
                return dirty;
            };
            // grad_out rows of the step, transposed: channel n = row of the K-major tile, reduction column gk
            auto fill_gout = [&](const uint4 &v) {
                const uint32_t w4[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const int n = gc * 8 + i;
                    const unsigned short h = (unsigned short)((i & 1) ? (w4[i >> 1] >> 16) : (w4[i >> 1] & 0xffffu));
                    dn::sts16(my_gt + (uint32_t)n * 128u + ((((uint32_t)gk >> 3) ^ ((uint32_t)n & 7u)) << 4) + (((uint32_t)gk & 7u) << 1), h);
                }
            };

            Smp cur[kMaxPass];
            load_samples(team, cur);
            uint4 gcur = load_gout(team);
            for (int step = team; step < nsteps; step += NT) {
                Smp nxt[kMaxPass];
                load_samples(step + NT, nxt);                    // next step's inputs are in flight during this one
                const uint4 gnxt = load_gout(step + NT);
                if (nuse > 0) dn::mbar_wait(&bar_empty[team], (nuse - 1) & 1);   // MMAs that read this slab retired
                // the mask of the previous use has been read by both issuers (their commits are in): clear it for the
                // use after this one -- ordered before that use's atomicOr through full[] -> empty[]
                if (tt == 0) s_dirty[2 * team + ((nuse + 1) & 1)] = 0;
                unscatter();
                uint32_t dirty = (dbg & 2) ? 0u : scatter(cur);
                dirty = __reduce_or_sync(0xffffffffu, dirty);
                if (lane == 0 && dirty) atomicOr(&s_dirty[2 * team + (nuse & 1)], dirty);
                if (g_role) fill_gout(gcur);
                dn::fence_async_smem();
                dn::mbar_arrive(&bar_full[team]);
                nuse++;
#pragma unroll
                for (int i = 0; i < kMaxPass; ++i) cur[i] = nxt[i];
                gcur = gnxt;
            }
            unit_bar();                                      // unit end: every MMA has retired
            unscatter();
            unit_bar();
        } else {
            // ================================ issuer warpgroups (even / odd tiles) ================================
            const int iw = team - NT, w4 = tw;
            uint32_t udirty = 0;                                  // tiles that hold data of this unit
#pragma unroll
            for (int i = 0; i < kMine; ++i)
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int e = 0; e < 16; ++e) acc[i][h][e] = 0.f;
            int t = 0;
            for (int step = 0; step < nsteps; ++step) {
                uint32_t par = 0;
#pragma unroll
                for (int i = 0; i < NT; ++i) if (i == t) { par = nfull[i] & 1u; nfull[i]++; }
                dn::mbar_wait(&bar_full[t], par);
                __syncwarp();
                const uint32_t mask = (dbg & 8) ? 0xfu : s_dirty[2 * t + par];   // the team clears it two uses later
                const uint64_t da0 = dn::desc_sw128(dn::s32(slab + t * kSlabBytes), 2048);
                const uint64_t db = dn::desc_sw128(dn::s32(gtile + t * 4096), 16);
                dn::wgmma_fence();
#pragma unroll
                for (int i = 0; i < kMine; ++i) {
                    const int tile = 2 * i + iw;
                    if (((mask >> tile) & 1u) && !(dbg & 1)) {        // warpgroup-uniform
#pragma unroll
                        for (int h = 0; h < 2; ++h)
                            dn::wgmma_m64n32_amn(acc[i][h], da0 + (uint64_t)((tile * kDnTileBytes + h * 2048) >> 4), db);
                    }
                }
                dn::wgmma_commit();
                dn::wgmma_wait0();
#pragma unroll
                for (int i = 0; i < kMine; ++i) { dn::fence_regs(acc[i][0]); dn::fence_regs(acc[i][1]); }
                udirty |= mask;
                __syncwarp();
                if (lane == 0) dn::mbar_arrive(&bar_empty[t]);
                if (++t == NT) t = 0;
            }
            unit_bar();                                           // unit end: the teams may clean their slabs
            // ---- flush: this warpgroup's touched tiles -> grad_value.  Warp w4 holds pixel rows 16 w4 .. 16 w4 + 15
            // of each 64-pixel half; they go through a 16 x 36 float transpose tile so that 8 lanes x 16 B cover one
            // 128 B (pixel, head) row of grad_value, 4 rows per instruction.
            if (!(dbg & (4 | 1))) {
                float *trw = tr + (iw * 4 + w4) * (kDnTransposeBytes / 4);
                const int sub = lane & 7;
#pragma unroll
                for (int i = 0; i < kMine; ++i) {
                    const int tile = 2 * i + iw;
                    if (!((udirty >> tile) & 1u)) continue;          // warpgroup-uniform
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
#pragma unroll
                        for (int j = 0; j < 4; ++j)
#pragma unroll
                            for (int hh = 0; hh < 2; ++hh)
                                *reinterpret_cast<float2 *>(trw + (8 * hh + (lane >> 2)) * 36 + 8 * j + 2 * (lane & 3)) =
                                    make_float2(acc[i][h][4 * j + 2 * hh], acc[i][h][4 * j + 2 * hh + 1]);
                        __syncwarp();
#pragma unroll
                        for (int q = 0; q < 4; ++q) {
                            const int rr = 4 * q + (lane >> 3);
                            const int row = tile * 128 + h * 64 + w4 * 16 + rr;
                            const float4 v = *reinterpret_cast<const float4 *>(trw + rr * 36 + sub * 4);
                            const bool nz = ((__float_as_uint(v.x) | __float_as_uint(v.y) | __float_as_uint(v.z) |
                                              __float_as_uint(v.w)) & 0x7fffffffu) != 0u;
                            if (nz && row < nb) {
                                float *gp = grad_value + (((long long)b * gv_S + s0 - gv_base + row) * M + m) * 32 + sub * 4;
                                red_add_v4(gp, v.x, v.y, v.z, v.w);
                            }
                        }
                        __syncwarp();
                    }
                }
            }
            unit_bar();
        }
    }
}

}  // namespace bevf

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
namespace bevf {

static long dense_env(const char *name, long dflt) {
    const char *e = getenv(name);
    return e ? strtol(e, nullptr, 0) : dflt;
}

// Bins of at most `cap` consecutive pixels over the levels l >= first with at most `max_pix` pixels: a level larger
// than a bin is cut into ceil(n / cap) bins, consecutive small levels share one (the kernel gives each level of a bin
// its own group of scatter threads).  Returns the mask of the covered levels, -1 for a bad shape, -2 if the table
// overflows.
static int plan_dense_bins(const int32_t *hw_host, int L, long max_pix, int cap, DenseBins &bins, long long *total,
                           int first = 0) {
    memset(&bins, 0, sizeof(bins));
    bins.L = L;
    long long start = 0;
    unsigned mask = 0;
    int open = -1;                                       // bin that may still take the next level
    for (int l = 0; l < L; ++l) {
        const int h = hw_host[2 * l], w = hw_host[2 * l + 1];
        if (h <= 0 || w <= 0 || h >= 32768 || w >= 32768) return -1;
        const long long n = (long long)h * w;
        bins.hl.h[l] = h; bins.hl.w[l] = w; bins.hl.start[l] = (int)start;
        if (l >= first && n <= max_pix) {
            if (n <= cap && open >= 0 && bins.n[open] + n <= cap && bins.nlev[open] < kDnBinLevels) {
                bins.lev[open][bins.nlev[open]++] = l;   // contiguous with the previous coarse level
                bins.n[open] += (int)n;
            } else {
                const int parts = (int)((n + cap - 1) / cap);
                if (bins.nbins + parts > kDnMaxBins) return -2;
                long long off = 0;
                for (int i = 0; i < parts; ++i) {
                    const int bi = bins.nbins++;
                    bins.s0[bi] = (int)(start + off);
                    bins.n[bi] = (int)((n - off) < cap ? (n - off) : cap);
                    bins.nlev[bi] = 1;
                    bins.lev[bi][0] = l;
                    off += bins.n[bi];
                }
                open = bins.nbins - 1;
            }
            mask |= 1u << l;
        } else {
            open = -1;
        }
        start += n;
    }
    *total = start;
    return (int)mask;
}

// Plans the bins from the HOST copy of the pyramid and launches the dense kernel for every level l >= first_level
// with at most `BEVF_DENSE_MAXPIX` pixels.  *handled = mask of the levels whose grad_value it produced (0: not
// applicable -- the caller then leaves every level to the reduction path).  need_mask != 0: launch only if the
// covered levels are exactly those (the mixed accumulation hands the dense kernel a whole suffix of the pyramid).
// grad_value, gv_S, gv_base: see msda_bwd_dense_tc.
int dense_coarse_backward(const char *who, const int64_t *hw_dev, const int64_t *ls_dev, const int32_t *hw_host,
                          const float *loc, const float *attn, const void *grad_out, float *grad_value,
                          const int32_t *map_range, int NB, int S, int M, int L, int P, cudaStream_t st,
                          unsigned *handled, HostLevels *host_levels, int first_level, unsigned need_mask,
                          int gv_S, int gv_base, int loc_level0) {
    *handled = 0;
    static const long max_pix = dense_env("BEVF_DENSE_MAXPIX", 8192);
    static const long tiles = dense_env("BEVF_DENSE_TILES", 4);
    static const long chunk = dense_env("BEVF_DENSE_CHUNK", 512);
    if ((P != 4 && P != 8) || L > kMaxLevels || NB <= 0 || max_pix <= 0) return 0;
    if (tiles != 4) return fail("%s: BEVF_DENSE_TILES must be 4", who);
    if (chunk < kDnK || chunk % kDnK) return fail("%s: BEVF_DENSE_CHUNK must be a positive multiple of 16", who);
    const int cap = (int)tiles * 128;
    DenseBins bins;
    long long start = 0;
    const int pm = plan_dense_bins(hw_host, L, max_pix, cap, bins, &start, first_level);
    if (pm == -1) return fail("%s: bad host level shape", who);
    if (pm == -2) return 0;                              // pyramid too large for the bin table
    const unsigned mask = (unsigned)pm;
    if (start != S) return fail("%s: host level shapes do not add up to S (%lld vs %lld)", who, start, S);
    if (mask == 0 || (need_mask != 0 && mask != need_mask)) return 0;
    static int sms = 0;
    if (sms == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    }
    static const long teams_env = dense_env("BEVF_DENSE_TEAMS", 0);
    const int teams = teams_env > 0 ? (int)teams_env : 3;     // 3: 12-15 % faster than 2 on the base SCA launch (H100)
    const size_t smem = 1024 + (size_t)teams * ((size_t)tiles * kDnTileBytes + 4096) + 8 * kDnTransposeBytes + 256;
    static const long dbg = dense_env("BEVF_DENSE_DEBUG", 0);       // development: 1 = no MMAs, 2 = no scatter, 4 = no flush, 8 = every tile counts as touched
    auto launch = [&](auto kern) -> int {
        // every instantiation has the same pointer type, so "configured" is remembered per kernel address
        static const void *configured[16];
        static int nconfigured = 0;
        static std::mutex mu;
        {
            std::lock_guard<std::mutex> lock(mu);
            bool seen = false;
            for (int i = 0; i < nconfigured; ++i) seen = seen || configured[i] == (const void *)kern;
            if (!seen) {
                if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
                    cudaGetLastError();
                    return fail("%s: cannot reserve shared memory for the dense backward", who);
                }
                if (nconfigured < 16) configured[nconfigured++] = (const void *)kern;
            }
        }
        kern<<<(unsigned)sms, 128 * teams + 256, smem, st>>>(bins, hw_dev, ls_dev, loc, attn, (const bf16 *)grad_out,
                                                           grad_value, map_range, NB, gv_S, gv_base, M, L, (int)chunk,
                                                           (int)dbg, loc_level0);
        return check_launch(who);
    };
    int e;
    if (teams < 1 || teams > 3) return fail("%s: BEVF_DENSE_TEAMS must be 1, 2 or 3", who);
    if (teams == 3) e = (P == 8) ? launch(msda_bwd_dense_tc<4, 8, 3>) : launch(msda_bwd_dense_tc<4, 4, 3>);
    else if (teams == 2) e = (P == 8) ? launch(msda_bwd_dense_tc<4, 8, 2>) : launch(msda_bwd_dense_tc<4, 4, 2>);
    else e = (P == 8) ? launch(msda_bwd_dense_tc<4, 8, 1>) : launch(msda_bwd_dense_tc<4, 4, 1>);
    if (e) return e;
    *handled = mask;
    *host_levels = bins.hl;
    return 0;
}

}  // namespace bevf

// Host-only: the bin plan the dense backward would use for this pyramid (tests / diagnostics; no device work).
extern "C" int bevf_msda_dense_plan(const int32_t *level_hw_host, int L, int max_pix, int tiles, int32_t *bins_out,
                                    int bins_cap, uint32_t *level_mask) {
    using namespace bevf;
    const char *who = "bevf_msda_dense_plan";
    if (!level_hw_host || !bins_out || !level_mask || L <= 0 || L > kMaxLevels || (tiles != 4 && tiles != 8 && tiles != 16))
        return -fail("%s: bad argument", who);
    DenseBins bins;
    long long total = 0;
    const int pm = plan_dense_bins(level_hw_host, L, max_pix, tiles * 128, bins, &total);
    if (pm == -1) return -fail("%s: bad host level shape", who);
    if (pm == -2) { *level_mask = 0; return 0; }
    if (bins.nbins > bins_cap) return -fail("%s: output too small", who);
    for (int i = 0; i < bins.nbins; ++i) {
        int32_t *o = bins_out + i * (3 + kDnBinLevels);
        o[0] = bins.s0[i]; o[1] = bins.n[i]; o[2] = bins.nlev[i];
        for (int j = 0; j < kDnBinLevels; ++j) o[3 + j] = j < bins.nlev[i] ? bins.lev[i][j] : -1;
    }
    *level_mask = (unsigned)pm;
    return bins.nbins;
}
