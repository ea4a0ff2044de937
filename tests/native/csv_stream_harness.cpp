// CPU harness for the streaming reader (lo_csv_stream_*, csrc/csv.inc): the same window bookkeeping
// (csv::StreamWindow), the same cut (csv::segment_last_end over the window's segments from their scanned start
// states) and the same per-window passes, with record indices and failure positions made absolute as the library does.
// The body arrives in the caller's pieces; each window is cut into segments of `seg` bytes.
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "csv_reader.cuh"

using namespace lo::csv;

namespace {

constexpr int64_t kNone = INT64_MAX;

struct Stream {
    StreamWindow w{0};
    int64_t seg = 256;
    std::vector<uint8_t> win;                        // w.cap bytes; [0, w.len) in use
    std::vector<std::vector<std::string>> cols;      // the cells of every kept record, header included
    int64_t info[6] = {0, 0, 0, 0, 6, -1};           // records, ncols, chars, fail_record, fail_kind, fail_pos
    bool done = false;
};

// the passes of one window [0, n) of s.win: starts from a scan of the maps, then (when cut < 0) the cut; returns the
// cut, or 0 when the window must grow
int64_t read_window(Stream &st, int64_t n, bool final) {
    const uint8_t *body = st.win.data();
    const int64_t nseg = (n + st.seg - 1) / st.seg;
    auto sb = [&](int64_t i) { return std::min(n, i * st.seg); };
    std::vector<uint32_t> starts(nseg);
    uint32_t m = kIdentityMap;
    for (int64_t i = 0; i < nseg; ++i) {
        starts[i] = map_apply(m, kStartRecord);
        m = map_compose(m, segment_map(body, sb(i), sb(i + 1)));
    }
    int64_t last = -1;
    for (int64_t i = 0; i < nseg && !final; ++i) last = std::max(last, segment_last_end(body, sb(i), sb(i + 1), starts[i]));
    const int64_t cut = st.w.cut(last, final);
    if (cut == 0) return 0;
    // [0, cut): the segments before the cut keep their start states
    const int64_t cs = (cut + st.seg - 1) / st.seg;
    auto cb = [&](int64_t i) { return std::min(cut, i * st.seg); };
    std::vector<Carry> carries(cs);
    Carry c = carry_zero();
    for (int64_t i = 0; i < cs; ++i) {
        carries[i] = c;
        NoVisit v;
        c = carry_combine(c, walk_segment(body, cut, cb(i), cb(i + 1), starts[i], carry_zero(), v));
    }
    const int64_t nrec = c.rec, rec0 = st.w.rec0;
    if (nrec == 0) {                                 // only breaks after the last record: the body's end
        st.w.advance(cut, 0, 0);
        return cut;
    }
    const int64_t ncols = rec0 == 0 ? c.first_col : st.w.ncols;
    int64_t fail_rec = kNone, short_rec = kNone;
    for (int64_t i = 0; i < cs; ++i) {
        ValidateVisit v{ncols, rec0};
        walk_segment(body, cut, cb(i), cb(i + 1), starts[i], carries[i], v);
        fail_rec = std::min(fail_rec, v.fail_rec);
        short_rec = std::min(short_rec, v.short_rec);
    }
    const int64_t kept = std::min(nrec, std::min(fail_rec, short_rec));
    const int64_t nlens = ncols * (kept + 1) + 1;
    std::vector<int64_t> lens(kept > 0 ? nlens : 1, 0);
    uint64_t key = UINT64_MAX;
    for (int64_t i = 0; i < cs; ++i) {
        LengthVisit v{lens.data(), ncols, kept, fail_rec};
        walk_segment(body, cut, cb(i), cb(i + 1), starts[i], carries[i], v);
        key = std::min(key, v.key);
    }
    if (kept > 0) {
        int64_t total = 0;
        for (int64_t i = 0; i < nlens; ++i) { const int64_t l = lens[i]; lens[i] = total; total += l; }
        std::vector<uint8_t> chars(total + 1);
        for (int64_t i = 0; i < cs; ++i) {
            ScatterVisit v{body, lens.data(), chars.data(), ncols, kept};
            walk_segment(body, cut, cb(i), cb(i + 1), starts[i], carries[i], v);
        }
        if (rec0 == 0) st.cols.assign(ncols, {});
        for (int64_t col = 0; col < ncols; ++col)
            for (int64_t r = 0; r < kept; ++r) {
                const int64_t a = lens[col * (kept + 1) + r], b = lens[col * (kept + 1) + r + 1];
                st.cols[col].emplace_back((const char *)chars.data() + a, b - a);
            }
        st.info[2] += total;
    }
    if (rec0 == 0) st.info[1] = kept > 0 ? ncols : 0;
    st.info[0] += kept;
    if (fail_rec != kNone && fail_rec <= short_rec) {
        static const int64_t kinds[4] = {3, 5, 4, 2};   // kFailUtf8, kFailTruncated, kFailNul, kFailFieldLimit
        st.info[3] = rec0 + fail_rec;
        st.info[4] = kinds[key & 3];
        st.info[5] = st.w.base + (int64_t)(key >> 2);
    } else if (short_rec != kNone) {
        st.info[3] = rec0 + short_rec;
        st.info[4] = 1;
    } else {
        st.info[3] = -1;
        st.info[4] = 0;
    }
    st.done = fail_rec != kNone || short_rec != kNone;
    st.w.advance(cut, nrec, ncols);
    return cut;
}

// lo_csv_stream_push: returns the bytes taken; at most one window is read
int64_t push(Stream &st, const uint8_t *bytes, int64_t n, bool last) {
    if (st.done) return n;
    StreamWindow &w = st.w;
    int64_t used = 0;
    for (;;) {
        const int64_t take = w.take(n - used);
        memcpy(st.win.data() + w.len, bytes + used, take);
        used += take;
        w.len += take;
        const bool final = last && used == n;
        if (!w.ready(final)) break;
        if (w.len == 0) { st.done = true; break; }
        const int64_t len = w.len;
        const int64_t cut = read_window(st, len, final);
        if (cut == 0) {
            w.grow();
            st.win.resize(w.cap);
            continue;
        }
        memmove(st.win.data(), st.win.data() + cut, len - cut);   // the tail (w.len is already len - cut)
        st.done = st.done || final;
        break;
    }
    return used;
}

}  // namespace

// pieces: npieces + 1 increasing positions from 0 to n (the body as pushed), then one zero-byte last push.  window:
// the starting capacity; seg: segment bytes inside a window.  info: records, ncols, chars, fail_record, fail_kind,
// fail_pos; offsets / chars in lo_csv_columns_host's layout.  Returns the number of pushes, -1 when offsets or
// chars are too small.
extern "C" int64_t csv_stream_read(const uint8_t *body, const int64_t *pieces, int64_t npieces, int64_t window,
                                   int64_t seg, int64_t *info, int64_t *offsets, int64_t offsets_cap, uint8_t *chars,
                                   int64_t chars_cap) {
    Stream st;
    st.w.cap = window;
    st.seg = seg;
    st.win.resize(window);
    int64_t pushes = 0;
    for (int64_t i = 0; i <= npieces && !st.done; ++i) {
        const bool last = i == npieces;
        const uint8_t *p = last ? body : body + pieces[i];
        const int64_t n = last ? 0 : pieces[i + 1] - pieces[i];
        int64_t off = 0;
        do {
            off += push(st, p + off, n - off, last);
            ++pushes;
        } while (!st.done && (off < n || last));
    }
    memcpy(info, st.info, sizeof st.info);
    const int64_t ncols = info[1], recs = info[0];
    if (recs == 0) return pushes;
    if (ncols * (recs + 1) > offsets_cap || info[2] > chars_cap) return -1;
    int64_t pos = 0;
    for (int64_t col = 0; col < ncols; ++col) {
        for (int64_t r = 0; r < recs; ++r) {
            offsets[col * (recs + 1) + r] = pos;
            const std::string &cell = st.cols[col][r];
            memcpy(chars + pos, cell.data(), cell.size());
            pos += (int64_t)cell.size();
        }
        offsets[col * (recs + 1) + recs] = pos;
    }
    return pushes;
}
