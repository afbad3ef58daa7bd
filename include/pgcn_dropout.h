/*
 * pgcn_dropout.h — C-ABI of the edge-dropout library (lib/libpgcn_dropout.so), sm_90a.
 *
 * Dropout on per-edge arrays whose mask is a pure function of the GLOBAL edge, so that every partition of a graph
 * draws the same mask, a backward recomputes it instead of storing it, and an fp64 oracle reproduces it bit for bit.
 * For an entry e with global row gi and global column gj, head h, 64-bit key and 32-bit call counter c:
 *
 *     (w0, w1, w2, w3) = Philox4x32-10(counter = (gi, gj, c, h >> 2), key = (key & 0xffffffff, key >> 32))
 *     u      = w[h & 3]
 *     keep   = u >= threshold               threshold = floor(p * 2^32)     (host, fp64, p in [0, 1))
 *     y[e,h] = keep ? x[e,h] * scale : x[e,h] * 0   (fp32)   scale = float32(1 / (1 - p))   (fp64 quotient, rounded once)
 *
 * Entries that repeat one (row, column) share their bit. NaN stays NaN. The plan library (pgcn_b200.h) is not
 * needed: the caller hands over each entry's (global row, global column).
 *
 * Conventions as pgcn_b200.h: extern "C", 0 or a negative status, never throws; asynchronous on the stream passed in.
 */
#ifndef PGCN_DROPOUT_H
#define PGCN_DROPOUT_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum pgcn_dropout_status {
    PGCN_DROPOUT_OK = 0,
    PGCN_DROPOUT_ERR_INVALID = -1,   /* null pointer or bad argument                  */
    PGCN_DROPOUT_ERR_CUDA = -2,      /* a CUDA runtime call or the launch failed       */
    PGCN_DROPOUT_ERR_NOGPU = -4      /* no CUDA device visible: there is no CPU path   */
} pgcn_dropout_status;

/* Version / build string (names the architecture, sm_90a). Never NULL. */
const char* pgcn_dropout_version(void);

/* Text of the last error of this library. Never NULL. */
const char* pgcn_dropout_last_error(void);

/*
 * y = mask(x) over nnz entries of `heads` values each (1, 2, 4 or 8), all DEVICE pointers:
 *   pairs   int32 [nnz, 2]   global (row, column) of each entry
 *   state   int64 [2]        (key, call counter), read on the device when the kernel runs, so that a CUDA graph that
 *                            advances the counter before this launch draws a new mask on every replay
 *   x, y    fp32 [nnz, heads], row-major; y may be x (in place), no other overlap
 * threshold and scale as above. Operands all aligned to 16 bytes take the vector instance, any other alignment the
 * scalar one; both give the same bits. nnz == 0 launches nothing.
 */
int pgcn_edge_dropout(const int32_t* pairs, int64_t nnz, int32_t heads, uint32_t threshold, float scale,
                      const int64_t* state, const float* x, float* y, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* PGCN_DROPOUT_H */
