// quotient.cuh — row-wise expression-program evaluator over extended cosets (the device side of evaluate_h).
#pragma once
#include "common.cuh"
#include "field.cuh"

namespace b200 {

// Operand encoding: bits 31..30 = kind (0 slot, 1 constant, 2 column load, 3 the previous instruction's result), bits 29..0 = index.
enum QSrcKind { QSRC_SLOT = 0, QSRC_CONST = 1, QSRC_LOAD = 2, QSRC_PREV = 3 };
enum QOp { QOP_ADD = 0, QOP_SUB = 1, QOP_MUL = 2, QOP_NEG = 3, QOP_DOUBLE = 4, QOP_SQUARE = 5, QOP_MOV = 6, QOP_MULADD = 7 };
static constexpr int Q_MAX_SLOTS = 256;
static constexpr uint32_t Q_NOSTORE = 0x80000000u;     // op_dst flag: the result is only read as PREV by the next instruction

struct QInstr { uint32_t op_dst; uint32_t a, b, c; };   // op_dst = op | (dst_slot << 8) | NOSTORE;  MULADD: a * b + c
struct QLoad { uint32_t column; uint32_t offset; };      // element offset already reduced mod 2^ext_k

// out[(idx << out_shift) + out_off] = program(columns[c][((idx + offset) mod N) << shift_c], constants) for idx < N = 2^ext_k, out_off < 2^out_shift
// (one coset part of a larger domain stores its rows interleaved, and reads the extended columns it is given in place with their stride 2^shift_c,
// from a base pointer already advanced to the part; 0, 0 is the dense layout).  h_col_shifts may be NULL (every shift 0).  h_* are host arrays;
// the program is staged through `ring` (common.cuh: StagingRing).
int quotient_eval_run(const Fr* const* h_col_ptrs /*device addresses*/, const uint32_t* h_col_shifts, size_t n_cols, uint32_t ext_k, const QLoad* h_loads,
                      size_t n_loads, const Fr* h_consts, size_t n_consts, const QInstr* h_prog, size_t n_instr, Fr* d_out, uint32_t out_shift, uint32_t out_off,
                      StagingRing& ring, cudaStream_t st);

}  // namespace b200
