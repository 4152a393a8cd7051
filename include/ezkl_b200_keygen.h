/*
 * ezkl_b200_keygen.h — key-generation entry points of libezkl_b200.so: the steps of create_keys (keygen_vk / keygen_pk) that are not
 * also steps of create_proof.  The types and conventions are those of ezkl_b200.h, which this header includes.
 */
#ifndef EZKL_B200_KEYGEN_H
#define EZKL_B200_KEYGEN_H

#include "ezkl_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- permutation argument: the sigma columns (halo2 plonk/permutation/keygen.rs, Assembly::build_vk / build_pk) ------------------
 * The mapping is the Assembly's after every copy constraint has been merged into its cycles: n_columns * 2^k pairs of uint32
 * (column, row), column-major, so cell (column j, row i) sits at mapping[2 * (j * 2^k + i)] (its column) and
 * mapping[2 * (j * 2^k + i) + 1] (its row).  The shim flattens halo2's `mapping: Vec<Vec<(usize, usize)>>` into this layout.
 * Sigma column j, row i = delta^c * omega^r where (c, r) is cell (j, i)'s entry: Fr in Montgomery form, fully reduced, so the bytes are
 * those of build_pk's `permutations` (halo2 computes them as a table of delta^j * omega^i followed by a gather).  omega = the domain's
 * n-th root of unity, delta = Fr::DELTA.  The library does not check that the mapping is a permutation (halo2 does not either); it only
 * needs every column < n_columns and every row < 2^k.
 * Both entry points: -1 for k > 28, and for a null pointer when n_columns > 0; 0 with no work when n_columns == 0.
 *
 * Host pointers: out[j] receives sigma column j (2^k elements).  Every cell is checked on the host before any device work: a cell
 * outside n_columns x 2^k returns -1 and writes nothing.  The mapping and the results are staged in column groups bounded by the
 * per-call scratch budget (B200_WS_BUDGET_MB, else derived from B200_WS_TOTAL_MB), which holds a group's 40 B per cell (8 B of mapping
 * and 32 B of result), so k = 26 and beyond need no more than one column at a time.  In a multi-device process the columns are dealt
 * over the devices, each staging its own columns over its own PCIe link.
 * Device pointers: sigma column j at d_out + 32 * j * out_stride bytes (out_stride >= 2^k elements, else -1); d_out must not overlap
 * d_mapping.  A cell outside n_columns x 2^k is written as zero; when `invalid` is non-NULL it receives the number of such cells and
 * the call synchronises its stream, otherwise the call only enqueues.  Runs on the device that owns d_out.
 * Device memory held beyond the caller's buffers: the table [delta^c, c < n_columns | omega^e, e < 2^ceil(k/2) | omega^(e 2^ceil(k/2)),
 * e < 2^floor(k/2)], 32 B per entry, in the thread's parameter ring (a slot up to 256 KiB, a reused device buffer above), 8 B for the
 * counter of invalid cells, and for the host-pointer form the staging of one column group. */
int b200_permutation_sigmas(const uint32_t* mapping, size_t n_columns, uint32_t k, const b200_fr* omega, const b200_fr* delta, b200_fr* const* out);
int b200_permutation_sigmas_dev(const void* d_mapping, size_t n_columns, uint32_t k, const b200_fr* omega, const b200_fr* delta, void* d_out, size_t out_stride,
                                uint64_t* invalid, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* EZKL_B200_KEYGEN_H */
