// expr.cu — temporal expressions (MDGPU_OP_EXPRESSION): arithmetic and math functions over the rows of other temporal properties of the plan
// (operators md_script_functions.inl:505-571, functions :576-603), evaluated per frame of a batch after its procedure properties.
//
// k_temporal_expr: one thread per (expression, frame of the batch, value). Element v of an array operand and the whole of a float operand are
// what value v of the result depends on, so every thread runs the postfix program on floats alone. Its operand stack lives in registers: the
// stack is only ever indexed through fully unrolled loops.
#include "common.cuh"
#include "kernels.h"

namespace mdg {

constexpr int EXPR_THREADS = 256;

// the reference calls the float function of libm; the transcendentals are evaluated in double and rounded once (see mdgpu.h)
__device__ __forceinline__ float expr_func1(uint32_t kind, float a) {
    switch (kind) {
    case MDGPU_EXPR_NEG: return -a;
    case MDGPU_EXPR_SQRT: return sqrtf(a);
    case MDGPU_EXPR_ABS: return fabsf(a);
    case MDGPU_EXPR_FLOOR: return floorf(a);
    case MDGPU_EXPR_CEIL: return ceilf(a);
    case MDGPU_EXPR_CBRT: return (float)cbrt((double)a);
    case MDGPU_EXPR_COS: return (float)cos((double)a);
    case MDGPU_EXPR_SIN: return (float)sin((double)a);
    case MDGPU_EXPR_ASIN: return (float)asin((double)a);
    case MDGPU_EXPR_ACOS: return (float)acos((double)a);
    case MDGPU_EXPR_ATAN: return (float)atan((double)a);
    case MDGPU_EXPR_LOG: return (float)log((double)a);
    case MDGPU_EXPR_EXP: return (float)exp((double)a);
    case MDGPU_EXPR_LOG2: return (float)log2((double)a);
    case MDGPU_EXPR_EXP2: return (float)exp2((double)a);
    default: return (float)log10((double)a);   // MDGPU_EXPR_LOG10
    }
}

__device__ __forceinline__ float expr_func2(uint32_t kind, float a, float b) {
    switch (kind) {
    case MDGPU_EXPR_ADD: return a + b;
    case MDGPU_EXPR_SUB: return a - b;
    case MDGPU_EXPR_MUL: return a * b;
    case MDGPU_EXPR_DIV: return a / b;
    case MDGPU_EXPR_MIN: return fminf(a, b);
    case MDGPU_EXPR_MAX: return fmaxf(a, b);
    case MDGPU_EXPR_ATAN2: return (float)atan2((double)a, (double)b);
    default: return (float)pow((double)a, (double)b);   // MDGPU_EXPR_POW
    }
}

__global__ void __launch_bounds__(EXPR_THREADS) k_temporal_expr(const ExprProg* progs, const ExprNode* nodes, uint32_t frame0, uint32_t B) {
    const ExprProg pg = progs[blockIdx.y];
    const uint32_t total = B * pg.len;
    for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < total; t += gridDim.x * blockDim.x) {
        const uint32_t f = t / pg.len, v = t - f * pg.len;
        const size_t row = (size_t)frame0 + f;
        float st[MDGPU_EXPR_MAX_DEPTH];
#pragma unroll
        for (int k = 0; k < MDGPU_EXPR_MAX_DEPTH; ++k) st[k] = 0.0f;
        int sp = 0;   // operands on the stack; the program was checked on the host: no underflow, no overflow, one result
        for (uint32_t i = 0; i < pg.num_nodes; ++i) {
            const ExprNode n = nodes[pg.first_node + i];
            float top = 0.0f, below = 0.0f;
#pragma unroll
            for (int k = 0; k < MDGPU_EXPR_MAX_DEPTH; ++k) { if (k == sp - 1) top = st[k]; if (k == sp - 2) below = st[k]; }
            float r; int at;
            if (n.kind == MDGPU_EXPR_CONST) { r = n.value; at = sp++; }
            else if (n.kind == MDGPU_EXPR_PROP) { r = n.src[row * n.src_len + (n.src_len == 1 ? 0u : v)]; at = sp++; }
            else if (n.kind >= MDGPU_EXPR_ATAN2 || (n.kind >= MDGPU_EXPR_ADD && n.kind <= MDGPU_EXPR_DIV)) { r = expr_func2(n.kind, below, top); at = --sp - 1; }
            else { r = expr_func1(n.kind, top); at = sp - 1; }
#pragma unroll
            for (int k = 0; k < MDGPU_EXPR_MAX_DEPTH; ++k) if (k == at) st[k] = r;
        }
        pg.out[row * pg.len + v] = st[0];
    }
}

void launch_temporal_expr(const ExprProg* d_progs, uint32_t n_progs, const ExprNode* d_nodes, uint32_t max_len, uint32_t frame0, int B, cudaStream_t s) {
    if (!n_progs || B <= 0) return;
    const uint32_t blocks = std::min<uint32_t>(((uint32_t)B * max_len + EXPR_THREADS - 1) / EXPR_THREADS, 1024u);
    k_temporal_expr<<<dim3(blocks, n_progs), EXPR_THREADS, 0, s>>>(d_progs, d_nodes, frame0, (uint32_t)B);
    note_launch("k_temporal_expr", s);
}

}  // namespace mdg
