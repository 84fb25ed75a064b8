/* oracle/ddstore_oracle.c -- TEST INFRASTRUCTURE, not product code.
 *
 * CPU restatement (plain C) of the reference's get() hot path, written from the reference's
 * semantics and checked against (a) the reference itself compiled verbatim
 * (oracle/_ref/libddstore_ref.so, built by oracle/Makefile) and (b) the committed golden
 * vectors under tests/golden/. Only tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline / --impl reference legs may load this; the product (libddstore_b200.so)
 * never does.
 *
 * Parity status: PINNED -- see tests/test_oracle.py (known answers from
 * /root/reference/test/demo.cxx:20-37, test/demo.py:37,55-56, test/test.py:144-159, the
 * sortedsearch tables, and byte-for-byte agreement with the verbatim-compiled reference on
 * seeded random worlds).
 *
 * Each function cites the reference file:line it follows.
 */
#include <stdint.h>
#include <string.h>

#define ORC_OK 0
#define ORC_ERR_DTYPE 1   /* "Invalid data type"       include/ddstore.hpp:202-203 */
#define ORC_ERR_START 2   /* "Invalid start on target" include/ddstore.hpp:210-211 */
#define ORC_ERR_COUNT 3   /* "Invalid count on target" include/ddstore.hpp:213-214 */
#define ORC_ERR_DISP 4    /* "Invalid disp"            include/ddstore.hpp:81-82   */

/* src/ddstore.cxx:5-17 -- first i>=1 with vec[i-1] <= num < vec[i]; 0 when num < vec[0] AND
 * when nothing matches (out of range falls back to rank 0 and is rejected later). */
int orc_sortedsearch(const long *vec, int n, long num) {
    int rtn = 0;
    for (int i = 1; i < n; i++) {
        if (vec[i - 1] <= num && num < vec[i]) {
            rtn = i;
            break;
        }
    }
    return rtn;
}

/* include/ddstore.hpp:75-89 -- all-gathered per-rank row counts -> INCLUSIVE running sum;
 * every rank must have passed the same disp (max-reduce compare, :78-82). */
int orc_lenlist(const long *nrows, const int *disp, int nranks, long *lenlist) {
    int max_disp = 0;
    for (int r = 0; r < nranks; r++)
        if (disp[r] > max_disp) max_disp = disp[r];
    for (int r = 0; r < nranks; r++)
        if (disp[r] != max_disp) return ORC_ERR_DISP; /* thrown on the ranks that differ */
    long sum = 0;
    for (int r = 0; r < nranks; r++) {
        sum += nrows[r];
        lenlist[r] = sum;
    }
    return ORC_OK;
}

/* include/ddstore.hpp:205-214 -- owner rank, first global row of the owner, the two checks */
int orc_locate(const long *lenlist, int nranks, long start, long count, int *target, long *offset) {
    int t = orc_sortedsearch(lenlist, nranks, start);
    long off = t > 0 ? lenlist[t - 1] : 0;
    *target = t;
    *offset = off;
    if (start < off) return ORC_ERR_START;
    /* Two intentional divergences from the reference (DESIGN.md section 5), whose `start + count > lenlist[t]` is UB
     * for both: a negative count, and a count for which start + count overflows, are "Invalid count on target".
     * start >= off >= 0 here, so lenlist[t] - start cannot overflow. */
    if (count < 0 || count > lenlist[t] - start) return ORC_ERR_COUNT;
    return ORC_OK;
}

/* include/ddstore.hpp:197-238 (method 0) -- one get(): itemsize check, locate, then the byte
 * copy MPI_Get performs: count*disp*itemsize bytes from base[target] + (start-offset) rows of
 * disp*itemsize bytes (window disp_unit, :58) into buf. */
int orc_get(const void *const *bases, const long *lenlist, int nranks, int disp, int itemsize, int req_itemsize,
            long start, long count, void *buf) {
    if (itemsize != req_itemsize) return ORC_ERR_DTYPE;
    int target;
    long offset;
    int rc = orc_locate(lenlist, nranks, start, count, &target, &offset);
    if (rc) return rc;
    size_t row = (size_t)disp * (size_t)itemsize;
    memcpy(buf, (const char *)bases[target] + (size_t)(start - offset) * row, (size_t)count * row);
    return ORC_OK;
}

/* The batched restatement (SURVEY.md section 8a, last paragraph): the loader's serial loop of
 * get() calls (examples/vae/distdataset.py:79-89) with each result appended to `out`.
 * out_offsets[i] = sum_{j<i} nbytes_j (B+1 entries). Stops at the first failing request like
 * the serial loop would (exception): returns its code and index in *bad. */
int orc_get_batch(const void *const *bases, const long *lenlist, int nranks, int disp, int itemsize,
                  int req_itemsize, const long *starts, const long *counts, long nreq, char *out,
                  long *out_offsets, long *bad) {
    size_t row = (size_t)disp * (size_t)itemsize;
    long pos = 0;
    for (long i = 0; i < nreq; i++) {
        if (out_offsets) out_offsets[i] = pos;
        int rc = orc_get(bases, lenlist, nranks, disp, itemsize, req_itemsize, starts[i], counts[i], out + pos);
        if (rc) {
            if (bad) *bad = i;
            return rc;
        }
        pos += (long)((size_t)counts[i] * row);
    }
    if (out_offsets) out_offsets[nreq] = pos;
    if (bad) *bad = -1;
    return ORC_OK;
}

/* The synthetic payload of SURVEY.md section 8d: element (global_row g, col c) of a variable with
 * seed s is the low `itemsize` bytes of splitmix64(s ^ (g*disp + c)). Host copy used to check the
 * device generator and to rebuild expected bytes for any index at full size. */
static inline uint64_t splitmix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ULL;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ULL;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBULL;
    return x ^ (x >> 31);
}

void orc_synth_rows(uint64_t seed, long first_global_row, long nrows, int disp, int itemsize, void *out) {
    unsigned char *p = (unsigned char *)out;
    for (long r = 0; r < nrows; r++)
        for (long c = 0; c < disp; c++) {
            uint64_t v = splitmix64(seed ^ (uint64_t)((first_global_row + r) * (long)disp + c));
            memcpy(p, &v, (size_t)itemsize); /* little-endian low bytes; itemsize <= 8 */
            p += itemsize;
        }
}
