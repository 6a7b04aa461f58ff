// rama.cu — VIAMD's Ramachandran density maps (src/components/ramachandran/ramachandran.cpp:1277-1370, rama_rep_compute_density) computed from the
// backbone angles that MDGPU_OP_BACKBONE_ANGLES left in HBM: every (phi, psi) of a frame range and of the segments of four residue classes adds 1 to a
// texel of a 512 x 512 map (one channel per class), then the map is blurred by three box passes along each axis (blur_density_gaussian :368-387).
//
// Buffers (all [512][512][4] = 1 Mi elements; element (x, y, c) of the map):
//   counts : u64, element at (x * 512 + y) * 4 + c — the layout the row passes of the blur walk. u64 because a texel of one class can receive more
//            than 2^32 samples over a long trajectory of a large protein; the map itself saturates at 2^24 (Convert).
//   buf[3] : float scratch. Row passes work on [x][y][c], column passes on [y][x][c], which is also VIAMD's density_tex layout: in both, element p of
//            the line of thread t = line * 4 + c sits at p * 2048 + t, so a warp reads and writes 128 contiguous bytes per step.
#include "common.cuh"
#include "kernels.h"

namespace mdg {

constexpr uint32_t RAMA_DIM = 512;
constexpr uint32_t RAMA_LINE_STRIDE = RAMA_DIM * 4;   // floats between consecutive positions of a line
constexpr uint32_t RAMA_NO_KEY = 0xffffffffu;

// Texel coordinate of w = u * 512: the reference's (uint32_t) truncates toward zero, so w in (-1, 0] — phi = -pi in float lands a hair below
// u = 0 — gives texel 0, and u = 1 (phi = pi in float) wraps to 0 through the mask. The clamp only keeps the conversion defined for w >= 2^32.
MDG_D uint32_t rama_texel(float w) { return (w > 0.0f ? (uint32_t)fminf(w, 4294967040.0f) : 0u) & (RAMA_DIM - 1); }

// The keyed lanes of the warp whose key equals this lane's (the set match.any.sync returns for them), from one ballot per key bit that differs
// within the warp: none when every keyed lane hit the same texel (a pile-up), at most the 20 bits of x, y and class. Lanes without a key take
// the first keyed lane's key so that they split no group, and are masked off by `keyed`. Ballots and reductions rather than match.any, because
// the kernels of this file are also executed on the CPU (tests/emul), which provides those. Called by the whole warp with keyed != 0.
MDG_D uint32_t rama_peers(uint32_t key, uint32_t keyed) {
    const uint32_t first = __shfl_sync(0xffffffffu, key, __ffs((int)keyed) - 1);
    const uint32_t k = key != RAMA_NO_KEY ? key : first;
    const uint32_t differ = __reduce_or_sync(0xffffffffu, k) & __reduce_or_sync(0xffffffffu, ~k);   // bits set in some lanes and clear in others
    uint32_t peers = keyed;
#pragma unroll
    for (int b = 0; b < 20; ++b) {
        if (!((differ >> b) & 1u)) continue;   // warp-uniform
        const uint32_t bit = (k >> b) & 1u, ones = __ballot_sync(0xffffffffu, bit);
        peers &= bit ? ones : ~ones;
    }
    return peers;
}

// One thread per (frame, class entry). A warp covers 32 consecutive items, so its trip count is uniform and every lane reaches the ballots:
// lanes that hit the same texel are merged and their leader adds the group's size (samples pile into the helix and sheet basins). The
// position (f, e) of a thread's item is advanced by the grid stride without dividing.
__global__ void __launch_bounds__(256) k_rama_scatter(RamaArgs a) {
    const uint64_t n = (uint64_t)a.frame_count * a.n_entries;
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    const uint64_t warp0 = (uint64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31u);
    const uint64_t i0 = warp0 + lane;
    uint32_t f = (uint32_t)(i0 / a.n_entries), e = (uint32_t)(i0 % a.n_entries);
    const uint32_t step_f = (uint32_t)(stride / a.n_entries), step_e = (uint32_t)(stride % a.n_entries);
    uint32_t cnt0 = 0, cnt1 = 0, cnt2 = 0, cnt3 = 0;
    for (uint64_t base = warp0; base < n; base += stride) {
        uint32_t key = RAMA_NO_KEY;
        if (f < a.frame_count) {
            const uint32_t fr = a.frame_beg + f;
            if ((a.mask[fr >> 6] >> (fr & 63u)) & 1ull) {
                const float2 ang = *reinterpret_cast<const float2*>(a.angles + ((size_t)fr * a.n_seg + a.seg[e]) * 2);
                if (!(ang.x == 0.0f && ang.y == 0.0f)) {   // segments without angles (chain ends) are skipped, as the reference does
                    const uint32_t c = (uint32_t)(e >= a.class_end[0]) + (uint32_t)(e >= a.class_end[1]) + (uint32_t)(e >= a.class_end[2]);
                    const float u = __fadd_rn(__fmul_rn(ang.x, a.scale), 0.5f), v = __fadd_rn(__fmul_rn(ang.y, a.scale), 0.5f);
                    const uint32_t x = rama_texel(__fmul_rn(u, (float)RAMA_DIM)), y = rama_texel(__fmul_rn(v, (float)RAMA_DIM));
                    key = ((x * RAMA_DIM + y) << 2) | c;
                    cnt0 += c == 0; cnt1 += c == 1; cnt2 += c == 2; cnt3 += c == 3;
                }
            }
        }
        const uint32_t keyed = __ballot_sync(0xffffffffu, key != RAMA_NO_KEY);
        if (keyed) {
            const uint32_t peers = rama_peers(key, keyed);
            if (key != RAMA_NO_KEY && lane == (uint32_t)(__ffs((int)peers) - 1)) atomicAdd(&a.counts[key], (unsigned long long)__popc(peers));
        }
        e += step_e; f += step_f;
        if (e >= a.n_entries) { e -= a.n_entries; ++f; }
    }
    const uint32_t s0 = __reduce_add_sync(0xffffffffu, cnt0), s1 = __reduce_add_sync(0xffffffffu, cnt1);
    const uint32_t s2 = __reduce_add_sync(0xffffffffu, cnt2), s3 = __reduce_add_sync(0xffffffffu, cnt3);
    if (lane == 0) {
        if (s0) atomicAdd(&a.samples[0], (unsigned long long)s0);
        if (s1) atomicAdd(&a.samples[1], (unsigned long long)s1);
        if (s2) atomicAdd(&a.samples[2], (unsigned long long)s2);
        if (s3) atomicAdd(&a.samples[3], (unsigned long long)s3);
    }
}

// The reference adds 1.0f per sample; a float stops growing at 2^24 (2^24 + 1 rounds back to 2^24), so the exact result is min(count, 2^24).
__global__ void k_rama_convert(const unsigned long long* __restrict__ counts, float* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= RAMA_DIM * RAMA_DIM * 4) return;
    const unsigned long long v = counts[i];
    out[i] = (float)(uint32_t)(v < (1ull << 24) ? v : (1ull << 24));
}

// One box pass of blur_rows_acc (:285-313) over one line: the window sum starts as in[-(k+1) .. k-1] (wrapped), then for every position
// acc = max(0, (acc - in[x-k-1]) + in[x+k]) and out[x] = acc * (1 / (2k+1)). The reference's three loops differ only in which index needs the
// wrap; masking both in every step reads the same elements. Loads are issued 16 positions ahead of the running sum, which stays in order.
MDG_D void rama_box_pass(const float* __restrict__ in, uint32_t in_step, float* __restrict__ out, int k) {
    const float scl = __fdiv_rn(1.0f, (float)(2 * k + 1));
    float acc = 0.0f;
    for (int x = -(k + 1); x < k; ++x) acc = __fadd_rn(acc, in[(uint32_t)(x & (int)(RAMA_DIM - 1)) * in_step]);
    for (int x0 = 0; x0 < (int)RAMA_DIM; x0 += 16) {
        float lo[16], hi[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            lo[j] = in[(uint32_t)((x0 + j - k - 1) & (int)(RAMA_DIM - 1)) * in_step];
            hi[j] = in[(uint32_t)((x0 + j + k) & (int)(RAMA_DIM - 1)) * in_step];
        }
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            acc = fmaxf(0.0f, __fadd_rn(__fsub_rn(acc, lo[j]), hi[j]));
            out[(size_t)(x0 + j) * RAMA_LINE_STRIDE] = __fmul_rn(acc, scl);
        }
    }
}

// Three passes over the lines of one direction, one thread per (line, channel): src -> t0 -> t1 -> dst. Each thread only touches its own line,
// so dst may be src. src is read either in the working layout (element p of thread t at p * 2048 + t) or transposed (line l, channel c at
// l * 2048 + p * 4 + c): the transpose of the reference between its row and column passes is a permutation, read here in place.
__global__ void __launch_bounds__(32) k_rama_blur_lines(const float* src, int src_transposed, float* t0, float* t1, float* dst, int k0, int k1, int k2) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= RAMA_DIM * 4) return;
    const uint32_t line = t >> 2, c = t & 3u;
    if (src_transposed) rama_box_pass(src + (size_t)line * RAMA_LINE_STRIDE + c, 4, t0 + t, k0);
    else rama_box_pass(src + t, RAMA_LINE_STRIDE, t0 + t, k0);
    rama_box_pass(t0 + t, RAMA_LINE_STRIDE, t1 + t, k1);
    rama_box_pass(t1 + t, RAMA_LINE_STRIDE, dst + t, k2);
}

void launch_rama_density(const RamaArgs& a, cudaStream_t s) {
    const size_t texels = (size_t)RAMA_DIM * RAMA_DIM * 4;
    cudaMemsetAsync(a.counts, 0, sizeof(unsigned long long) * texels, s);
    cudaMemsetAsync(a.samples, 0, sizeof(unsigned long long) * 4, s);
    const uint64_t n = (uint64_t)a.frame_count * a.n_entries;
    if (n) {
        const uint64_t want = (n + 255) / 256, cap = (uint64_t)(a.sm_count > 0 ? a.sm_count : 132) * 8;
        const unsigned blocks = (unsigned)(want < cap ? want : cap);
        k_rama_scatter<<<blocks, 256, 0, s>>>(a);
        note_launch("k_rama_scatter", s);
    }
    k_rama_convert<<<(unsigned)((texels + 255) / 256), 256, 0, s>>>(a.counts, a.buf[0]);
    note_launch("k_rama_convert", s);
    // rows (along x, counts layout [x][y][c]): buf0 -> buf1 -> buf2 -> buf0; columns (along y): buf0 read transposed -> buf1 -> buf2 -> buf1 = [y][x][c]
    k_rama_blur_lines<<<RAMA_DIM * 4 / 32, 32, 0, s>>>(a.buf[0], 0, a.buf[1], a.buf[2], a.buf[0], a.box[0], a.box[1], a.box[2]);
    note_launch("k_rama_blur_lines", s);
    k_rama_blur_lines<<<RAMA_DIM * 4 / 32, 32, 0, s>>>(a.buf[0], 1, a.buf[1], a.buf[2], a.buf[1], a.box[0], a.box[1], a.box[2]);
    note_launch("k_rama_blur_lines", s);
}

}  // namespace mdg
