// tests/cpp/pad_layout_check.cpp -- the layout of a padded batch, checked on the host.
//
// The padded gather (dds_gather_kernel with PAD) walks the padded source space [0, nreq * slot) in segments of
// ddsk_fixed_seg_bytes(...) bytes. Inside a segment it copies each slot's payload in pieces of at most CH bytes and fills
// the slot's padding, both as ddsk_pad_cut (kernels.h) says. This program replays that cutting for many shapes -- raw
// and converting position maps, every itemsize, empty and truncated requests, several grid sizes, and one batch whose
// output passes 4 GiB -- and checks that every output byte of [0, nreq * slot_out) is written exactly once, as payload
// or as padding, that nothing outside it is written, and that no cut splits an element. Exit status 0: all shapes hold.
#include <stdint.h>
#include <stdio.h>

#include <algorithm>
#include <random>
#include <vector>

#include "kernels.h"

namespace {

constexpr int64_t kCH = 4096; // chunk of the padded gather's geometry (12 warps x 4 stages x 4096 bytes)

struct Interval {
    int64_t lo, hi;
    bool pad;
};

struct Shape {
    int64_t nreq, max_rows, row_bytes, nwarps;
    int in_log2, out_log2; // source -> output position map (0 / 0: raw)
    int in_el, out_el;     // source / output element size in bytes
};

int g_fail = 0;

void failf(const Shape &s, const char *what, int64_t a, int64_t b) {
    if (g_fail++ < 20)
        fprintf(stderr, "FAIL %s (%lld, %lld): nreq %lld max_rows %lld row_bytes %lld nwarps %lld map %d->%d\n", what,
                (long long)a, (long long)b, (long long)s.nreq, (long long)s.max_rows, (long long)s.row_bytes,
                (long long)s.nwarps, s.in_log2, s.out_log2);
}

// payload bytes of every request: min(count, max_rows) * row_bytes, 0 for an invalid one
std::vector<int64_t> payloads(const Shape &s, std::mt19937_64 &rng) {
    std::vector<int64_t> p((size_t)s.nreq);
    for (auto &x : p) {
        const int64_t count = (int64_t)(rng() % (uint64_t)(2 * s.max_rows + 2));
        const bool invalid = rng() % 16 == 0;
        x = invalid ? 0 : std::min(count, s.max_rows) * s.row_bytes;
    }
    return p;
}

void check(const Shape &s, const std::vector<int64_t> &payload) {
    const int64_t slot = s.max_rows * s.row_bytes;
    const int64_t T = s.nreq * slot;
    const int64_t out_total = (T >> s.in_log2) << s.out_log2;
    std::vector<Interval> w;
    if (T > 0) {
        const int64_t seg = ddsk_fixed_seg_bytes(T, slot, s.nwarps, 1, kCH);
        if (seg <= 0 || (seg % slot != 0 && seg % kCH != 0)) failf(s, "segment size (whole slots or whole chunks)", seg, slot);
        for (int64_t sp = 0; sp < T; sp += seg) {
            const int64_t se = std::min(T, sp + seg);
            const int64_t i_end = std::min(s.nreq, (se + slot - 1) / slot);
            for (int64_t i = sp / slot; i < i_end; i++) {
                const ddsk_pad_cut_t c = ddsk_pad_cut(i, payload[(size_t)i], slot, std::max<int64_t>(sp - i * slot, 0),
                                                      std::min(se - i * slot, slot), s.in_log2, s.out_log2);
                // the walk copies the payload part in pieces of at most CH source bytes
                for (int64_t p = c.pay_src; p < c.pay_src + c.pay_len; p += kCH) {
                    const int64_t n = std::min(kCH, c.pay_src + c.pay_len - p);
                    if (p % s.in_el || n % s.in_el) failf(s, "payload piece cuts a source element", p, n);
                    const int64_t d = (p >> s.in_log2) << s.out_log2;
                    if (p == c.pay_src && d != c.pay_dst) failf(s, "payload destination", d, c.pay_dst);
                    w.push_back({d, d + ((n >> s.in_log2) << s.out_log2), false});
                }
                if (c.pad_len > 0) {
                    if (c.pad_dst % s.out_el || c.pad_len % s.out_el) failf(s, "padding cuts an output element", c.pad_dst, c.pad_len);
                    w.push_back({c.pad_dst, c.pad_dst + c.pad_len, true});
                }
            }
        }
    }
    std::sort(w.begin(), w.end(), [](const Interval &a, const Interval &b) { return a.lo < b.lo; });
    int64_t at = 0;
    for (const Interval &x : w) {
        if (x.hi <= x.lo) failf(s, "empty write", x.lo, x.hi);
        if (x.lo != at) failf(s, x.lo < at ? "byte written twice" : "byte never written", at, x.lo);
        at = std::max(at, x.hi);
    }
    if (at != out_total) failf(s, "end of the writes vs the padded size", at, out_total);
    // every slot: payload then padding, exactly at its place in the output
    int64_t pay = 0, pad = 0;
    for (const Interval &x : w) (x.pad ? pad : pay) += x.hi - x.lo;
    int64_t want_pay = 0;
    for (int64_t p : payload) want_pay += (p >> s.in_log2) << s.out_log2;
    if (pay != want_pay || pay + pad != out_total) failf(s, "payload / padding byte counts", pay, want_pay);
}

} // namespace

int main() {
    std::mt19937_64 rng(12345);
    int shapes = 0;
    // raw batches: itemsize x row width, the grid sizes of 132 SMs at one and two CTAs per SM, and a tiny grid
    const int64_t nreqs[] = {0, 1, 31, 32, 33, 1023, 1024, 1025};
    const int64_t max_rows[] = {0, 1, 3, 64, 1000};
    const int64_t nwarps[] = {132 * 12, 2 * 132 * 12, 12};
    for (int el = 1; el <= 8; el *= 2)
        for (int64_t disp : {1, 3, 12, 37, 4097 / el})
            for (int64_t mr : max_rows)
                for (int64_t nr : nreqs)
                    for (int64_t nw : nwarps) {
                        const Shape s{nr, mr, disp * el, nw, 0, 0, el, el};
                        check(s, payloads(s, rng));
                        shapes++;
                    }
    // converting batches: (source itemsize, output itemsize) of every DDS_CVT_* code
    const int cv[][2] = {{2, 1}, {3, 2}, {0, 1}, {0, 2}, {2, 2}};
    for (auto &c : cv)
        for (int64_t disp : {1, 3, 80, 1025})
            for (int64_t mr : max_rows)
                for (int64_t nr : nreqs) {
                    const Shape s{nr, mr, disp << c[0], 132 * 12, c[0], c[1], 1 << c[0], 1 << c[1]};
                    check(s, payloads(s, rng));
                    shapes++;
                }
    // slots around CH and of several MiB
    for (int64_t rb : {4, 8})
        for (int64_t mr : {kCH / rb - 1, kCH / rb, kCH / rb + 1, (int64_t)(3 << 20) / rb})
            for (int64_t nr : {1, 33, 200}) {
                const Shape s{nr, mr, rb, 132 * 12, 0, 0, (int)rb, (int)rb};
                check(s, payloads(s, rng));
                shapes++;
            }
    // one batch whose padded output passes 4 GiB: 65536 slots of 16400 float32 rows (65600 bytes each)
    {
        const Shape s{65536, 16400, 4, 132 * 12, 0, 0, 4, 4};
        check(s, payloads(s, rng));
        shapes++;
    }
    if (g_fail) {
        fprintf(stderr, "%d failures\n", g_fail);
        return 1;
    }
    printf("pad layout ok: %d shapes\n", shapes);
    return 0;
}
