// CPU harness for learningorchestra_b200/csrc/csv_reader.cuh: the device reader's passes (csv.inc) run here on
// segments of the caller's choosing — maps composed by an exclusive scan, carries combined by an exclusive scan, then
// every segment re-walked from its scanned state — so the decomposition itself is checked, not just the rules.
#include <stdint.h>

#include <algorithm>
#include <vector>

#include "csv_reader.cuh"

using namespace lo::csv;

// bounds: nseg + 1 increasing positions from 0 to n.  info: records, ncols, chars, fail_record, fail_kind, fail_pos.
// offsets: room for ncols * (records + 1) entries, chars: room for n bytes.  Returns 0, or -1 when offsets is too small.
extern "C" int csv_read(const uint8_t *body, int64_t n, const int64_t *bounds, int64_t nseg, int64_t *info,
                        int64_t *offsets, int64_t offsets_cap, uint8_t *chars) {
    info[0] = info[1] = info[2] = 0;
    info[3] = 0;
    info[4] = 6;   // LO_CSV_EMPTY
    info[5] = -1;
    if (n == 0) return 0;
    std::vector<uint32_t> starts(nseg);
    std::vector<Carry> carries(nseg);
    uint32_t m = kIdentityMap;
    for (int64_t i = 0; i < nseg; ++i) {
        starts[i] = map_apply(m, kStartRecord);
        m = map_compose(m, segment_map(body, bounds[i], bounds[i + 1]));
    }
    Carry c = carry_zero();
    for (int64_t i = 0; i < nseg; ++i) {
        carries[i] = c;
        NoVisit v;
        c = carry_combine(c, walk_segment(body, n, bounds[i], bounds[i + 1], starts[i], carry_zero(), v));
    }
    const int64_t nrec = c.rec;
    if (nrec == 0) return 0;
    const int64_t ncols = c.first_col;
    int64_t fail_rec = INT64_MAX, short_rec = INT64_MAX;
    for (int64_t i = 0; i < nseg; ++i) {
        ValidateVisit v{ncols};
        walk_segment(body, n, bounds[i], bounds[i + 1], starts[i], carries[i], v);
        fail_rec = std::min(fail_rec, v.fail_rec);
        short_rec = std::min(short_rec, v.short_rec);
    }
    const int64_t kept = std::min(nrec, std::min(fail_rec, short_rec));
    const int64_t nlens = ncols * (kept + 1) + 1;
    std::vector<int64_t> lens(kept > 0 ? nlens : 1, 0);
    uint64_t key = UINT64_MAX;
    for (int64_t i = 0; i < nseg; ++i) {
        LengthVisit v{lens.data(), ncols, kept, fail_rec};
        walk_segment(body, n, bounds[i], bounds[i + 1], starts[i], carries[i], v);
        key = std::min(key, v.key);
    }
    int64_t total = 0;
    if (kept > 0) {
        if (nlens - 1 > offsets_cap) return -1;
        for (int64_t i = 0; i < nlens; ++i) { const int64_t l = lens[i]; lens[i] = total; total += l; }
        for (int64_t i = 0; i < nseg; ++i) {
            ScatterVisit v{body, lens.data(), chars, ncols, kept};
            walk_segment(body, n, bounds[i], bounds[i + 1], starts[i], carries[i], v);
        }
        std::copy(lens.begin(), lens.end() - 1, offsets);
        total = lens[nlens - 1];
    }
    info[0] = kept;
    info[1] = kept > 0 ? ncols : 0;
    info[2] = total;
    if (fail_rec != INT64_MAX && fail_rec <= short_rec) {
        static const int64_t kinds[4] = {3, 5, 4, 2};   // kFailUtf8, kFailTruncated, kFailNul, kFailFieldLimit
        info[3] = fail_rec;
        info[4] = kinds[key & 3];
        info[5] = (int64_t)(key >> 2);
    } else if (short_rec != INT64_MAX) {
        info[3] = short_rec;
        info[4] = 1;
    } else {
        info[3] = -1;
        info[4] = 0;
    }
    return 0;
}
