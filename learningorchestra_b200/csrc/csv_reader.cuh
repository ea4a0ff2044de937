// csv_reader.cuh — the CSV rules of the reference's upload reader, byte by byte, for the device reader (csv.inc) and
// the g++ harnesses (tests/native/csv_harness.cpp, csv_stream_harness.cpp).  __host__ __device__, no CUDA runtime calls.
//
// The reference reads an upload with
//     csv.reader(codecs.iterdecode(response.iter_lines(), "utf-8"), delimiter=",", quotechar='"')
// (database_api_image/database.py:110-137).  Restated on bytes:
//   * lines end at every run of '\r' / '\n' bytes; empty lines never reach the csv module, so a run of breaks is ONE
//     end of line (the first byte of the run), the rest of the run is skipped;
//   * the reader is CPython's _csv state machine with the default dialect (strict=False, no escapechar, doublequote):
//     START_RECORD, START_FIELD, IN_FIELD, IN_QUOTED_FIELD, QUOTE_IN_QUOTED_FIELD; a quote opens a field only at its
//     start, "" inside quotes is one quote, text after a closing quote is appended, a line end inside quotes is
//     dropped, an unterminated quote at EOF ends the record with what it has;
//   * a field holds at most kFieldLimit code points; UTF-8 is decoded strictly line by line; Python 3.7's _csv (the
//     reference image) rejects NUL.
//
// Parallel form: the body is cut into segments.  The transition map of a segment (end state for each of the 5 start
// states, 3 bits each) composes associatively, so a scan of the maps gives every segment its start state.  A second
// scan over CsvCarry (records ended, last line break, field index in the record, bytes / code points of the open
// field) gives every segment what it needs to know about the bytes before it.  Then any pass re-walks its segment
// with walk_segment() and sees, at every byte, the record, column and in-field offset it belongs to.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define LO_CSV_HD __host__ __device__ __forceinline__
#else
#define LO_CSV_HD inline
#endif

namespace lo {
namespace csv {

enum : uint32_t { kStartRecord = 0, kStartField = 1, kInField = 2, kInQuoted = 3, kQuoteInQuoted = 4 };
constexpr int kStates = 5;
constexpr int64_t kFieldLimit = 131072;        // csv.field_size_limit() default, in code points

// byte classes: a line end is the FIRST byte of a run of '\r' / '\n'; the others of the run are skipped
enum : uint32_t { kOther = 0, kQuote = 1, kComma = 2, kEol = 3, kSkip = 4 };

LO_CSV_HD bool is_break(uint32_t b) { return b == '\r' || b == '\n'; }

LO_CSV_HD uint32_t byte_class(uint32_t b, int32_t prev /* byte before, -1 at the start of the body */) {
    if (is_break(b)) return (prev == '\r' || prev == '\n') ? kSkip : kEol;
    return b == '"' ? kQuote : b == ',' ? kComma : kOther;
}

// what a step does besides changing state
enum : uint32_t { kKeep = 1, kSave = 2, kEnd = 4 };

// (state, class) -> next state | actions << 4.  Rows: states; columns: kOther, kQuote, kComma, kEol, kSkip.
LO_CSV_HD uint32_t step(uint32_t s, uint32_t cls) {
    // packed as 5 x 5 entries of one byte each would need a table in memory; the switch compiles to selects
    switch (s) {
        case kStartRecord:
            return cls == kOther ? (kInField | kKeep << 4) : cls == kQuote ? kInQuoted
                 : cls == kComma ? (kStartField | kSave << 4) : kStartRecord;
        case kStartField:
            return cls == kOther ? (kInField | kKeep << 4) : cls == kQuote ? kInQuoted
                 : cls == kComma ? (kStartField | kSave << 4) : cls == kEol ? (kStartRecord | (kSave | kEnd) << 4) : kStartField;
        case kInField:
            return cls == kOther || cls == kQuote ? (kInField | kKeep << 4)
                 : cls == kComma ? (kStartField | kSave << 4) : cls == kEol ? (kStartRecord | (kSave | kEnd) << 4) : kInField;
        case kInQuoted:
            return cls == kOther || cls == kComma ? (kInQuoted | kKeep << 4) : cls == kQuote ? kQuoteInQuoted : kInQuoted;
        default:  // kQuoteInQuoted
            return cls == kOther ? (kInField | kKeep << 4) : cls == kQuote ? (kInQuoted | kKeep << 4)
                 : cls == kComma ? (kStartField | kSave << 4) : cls == kEol ? (kStartRecord | (kSave | kEnd) << 4) : kQuoteInQuoted;
    }
}

// ---- transition maps: bits [3s, 3s+3) = end state for start state s ----------------------------------------------
constexpr uint32_t kIdentityMap = 0u | 1u << 3 | 2u << 6 | 3u << 9 | 4u << 12;

LO_CSV_HD uint32_t map_apply(uint32_t m, uint32_t s) { return (m >> (3 * s)) & 7u; }

// `a` then `b` (associative, not commutative)
LO_CSV_HD uint32_t map_compose(uint32_t a, uint32_t b) {
    uint32_t r = 0;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (uint32_t s = 0; s < kStates; ++s) r |= map_apply(b, map_apply(a, s)) << (3 * s);
    return r;
}

struct MapCompose {
    LO_CSV_HD uint32_t operator()(uint32_t a, uint32_t b) const { return map_compose(a, b); }
};

// ---- UTF-8 (CPython's strict decoder) ------------------------------------------------------------------------------
LO_CSV_HD bool is_cont(uint32_t b) { return (b & 0xC0u) == 0x80u; }

// sequence length of a valid lead byte, 0 for bytes no sequence starts with (continuations, C0, C1, F5..FF)
LO_CSV_HD int lead_len(uint32_t b) {
    return b < 0x80u ? 1 : b < 0xC2u ? 0 : b < 0xE0u ? 2 : b < 0xF0u ? 3 : b < 0xF5u ? 4 : 0;
}

// the second byte's range depends on the lead (no overlongs, no surrogates, nothing above U+10FFFF)
LO_CSV_HD bool second_ok(uint32_t lead, uint32_t b) {
    if (lead == 0xE0u) return b >= 0xA0u && b <= 0xBFu;
    if (lead == 0xEDu) return b >= 0x80u && b <= 0x9Fu;
    if (lead == 0xF0u) return b >= 0x90u && b <= 0xBFu;
    if (lead == 0xF4u) return b >= 0x80u && b <= 0x8Fu;
    return is_cont(b);
}

enum : uint32_t { kUtf8Ok = 0, kUtf8Bad = 1, kUtf8Truncated = 2 };

// Byte p >= 0x80 of the body: kUtf8Bad when the decoder rejects it (its line raises UnicodeDecodeError);
// kUtf8Truncated when p leads a sequence that is valid so far but its line (or the body) ends before it is complete —
// the incremental decoder would join it with the next line, which the device reader does not reproduce.
LO_CSV_HD uint32_t utf8_check(const uint8_t *body, int64_t n, int64_t p) {
    const uint32_t b = body[p];
    if (is_cont(b)) {               // valid only inside the sequence of a lead at most 3 bytes back
        int64_t q = p - 1;
        while (q >= 0 && q > p - 4 && is_cont(body[q])) --q;
        if (q < 0 || q <= p - 4) return kUtf8Bad;
        const int L = lead_len(body[q]);
        return (L > 1 && p - q < L && second_ok(body[q], body[q + 1])) ? kUtf8Ok : kUtf8Bad;
    }
    const int L = lead_len(b);
    if (L == 0) return kUtf8Bad;
    for (int i = 1; i < L; ++i) {
        if (p + i >= n || is_break(body[p + i])) return kUtf8Truncated;
        const uint32_t c = body[p + i];
        if (i == 1 ? !second_ok(b, c) : !is_cont(c)) return kUtf8Bad;   // the bad byte is not a continuation: flagged here
    }
    return kUtf8Ok;
}

// ---- failures -------------------------------------------------------------------------------------------------------
// Failure kinds in the order the reference meets them at one position: a line's decode error (or truncated sequence)
// is raised when the line is fetched, before any of its characters; NUL is rejected before a character is added.
enum : uint32_t { kFailUtf8 = 0, kFailTruncated = 1, kFailNul = 2, kFailFieldLimit = 3 };
// key = position * 4 + kind; the smallest key is the failure the reference raises first
LO_CSV_HD uint64_t fail_key(int64_t pos, uint32_t kind) { return (uint64_t)pos * 4u + kind; }

// ---- what a segment carries to the next ----------------------------------------------------------------------------
enum : uint32_t { kHasEnd = 1, kHasSave = 2 };
struct Carry {
    int64_t  rec;        // record ends (before this point)
    int64_t  lastbrk;    // position of the last '\r' / '\n' byte, -1 if none
    int64_t  col;        // fields saved since the last record end (= column of the open field)
    int64_t  fbytes;     // bytes kept in the open field
    int64_t  fcps;       // code points kept in the open field
    int64_t  first_col;  // fields of the first record that ended (valid when kHasEnd)
    uint32_t flags;
    uint32_t pad;
};

LO_CSV_HD Carry carry_zero() { return Carry{0, -1, 0, 0, 0, 0, 0, 0}; }

// `a` then `b`
LO_CSV_HD Carry carry_combine(const Carry &a, const Carry &b) {
    Carry r;
    r.rec = a.rec + b.rec;
    r.lastbrk = a.lastbrk > b.lastbrk ? a.lastbrk : b.lastbrk;
    r.col = (b.flags & kHasEnd) ? b.col : a.col + b.col;
    r.fbytes = (b.flags & kHasSave) ? b.fbytes : a.fbytes + b.fbytes;
    r.fcps = (b.flags & kHasSave) ? b.fcps : a.fcps + b.fcps;
    r.first_col = (a.flags & kHasEnd) ? a.first_col : (b.flags & kHasEnd) ? a.col + b.first_col : 0;
    r.flags = a.flags | b.flags;
    r.pad = 0;
    return r;
}

struct CarryCombine {
    LO_CSV_HD Carry operator()(const Carry &a, const Carry &b) const { return carry_combine(a, b); }
};

// ---- one segment ----------------------------------------------------------------------------------------------------
// Transition map of bytes [b, e).
LO_CSV_HD uint32_t segment_map(const uint8_t *body, int64_t b, int64_t e) {
    uint32_t st[kStates] = {0, 1, 2, 3, 4};
    int32_t prev = b > 0 ? (int32_t)body[b - 1] : -1;
    for (int64_t p = b; p < e; ++p) {
        const uint32_t cls = byte_class(body[p], prev);
        prev = body[p];
        for (int s = 0; s < kStates; ++s) st[s] = step(st[s], cls) & 7u;
    }
    return st[0] | st[1] << 3 | st[2] << 6 | st[3] << 9 | st[4] << 12;
}

template <class V>
LO_CSV_HD void apply_ends(uint32_t act, Carry &c, V &v) {
    if (act & kSave) {
        v.save(c);
        ++c.col;
        c.fbytes = 0;
        c.fcps = 0;
        c.flags |= kHasSave;
    }
    if (act & kEnd) {
        v.end(c);
        if (!(c.flags & kHasEnd)) c.first_col = c.col;
        ++c.rec;
        c.col = 0;
        c.flags |= kHasEnd;
    }
}

// Walks bytes [b, e) from state `s` with everything before b summarised in `c`, calling
//   v.keep(p, c)        a kept byte (c.col / c.rec / c.fbytes: its field and offset in it)
//   v.save(c)           a field ends (c.col its column, c.fbytes its length, c.rec its record)
//   v.end(c)            a record ends (c.rec its index, c.col its number of fields)
//   v.fail(c, key)      a failure (fail_key) inside record c.rec
// and, when e == n, the end of the body.  Returns the carry after e.
template <class V>
LO_CSV_HD Carry walk_segment(const uint8_t *body, int64_t n, int64_t b, int64_t e, uint32_t s, Carry c, V &v) {
    int32_t prev = b > 0 ? (int32_t)body[b - 1] : -1;
    for (int64_t p = b; p < e; ++p) {
        const uint32_t byte = body[p];
        const uint32_t cls = byte_class(byte, prev);
        prev = (int32_t)byte;
        if (cls >= kEol) c.lastbrk = p;
        if (byte >= 0x80u) {
            const uint32_t u = utf8_check(body, n, p);
            if (u != kUtf8Ok) v.fail(c, fail_key(c.lastbrk + 1, u == kUtf8Bad ? kFailUtf8 : kFailTruncated));
        } else if (byte == 0) {
            v.fail(c, fail_key(p, kFailNul));
        }
        const uint32_t t = step(s, cls);
        s = t & 7u;
        const uint32_t act = t >> 4;
        if (act & kKeep) {
            if (!is_cont(byte)) {
                if (c.fcps >= kFieldLimit) v.fail(c, fail_key(p, kFailFieldLimit));
                ++c.fcps;
            }
            v.keep(p, c);
            ++c.fbytes;
        }
        apply_ends(act, c, v);
    }
    if (e == n && n > 0) {
        // the reader processes an end of line after the last line too, terminated or not; then an unterminated quote
        // ends the record with what it has
        if (!is_break(body[n - 1])) {
            const uint32_t t = step(s, kEol);
            s = t & 7u;
            apply_ends(t >> 4, c, v);
        }
        if (s == kInQuoted) apply_ends(kSave | kEnd, c, v);
    }
    return c;
}

// ---- the passes' visitors -------------------------------------------------------------------------------------------
struct NoVisit {
    LO_CSV_HD void keep(int64_t, const Carry &) {}
    LO_CSV_HD void save(const Carry &) {}
    LO_CSV_HD void end(const Carry &) {}
    LO_CSV_HD void fail(const Carry &, uint64_t) {}
};

// first record with a parse failure, first data record with fewer than ncols fields; rec0 = records before the bytes
// walked (0 for a whole body, so record 0 is the header)
struct ValidateVisit {
    int64_t ncols;
    int64_t rec0 = 0;
    int64_t fail_rec = INT64_MAX, short_rec = INT64_MAX;
    LO_CSV_HD void keep(int64_t, const Carry &) {}
    LO_CSV_HD void save(const Carry &) {}
    LO_CSV_HD void end(const Carry &c) { if (rec0 + c.rec > 0 && c.col < ncols && c.rec < short_rec) short_rec = c.rec; }
    LO_CSV_HD void fail(const Carry &c, uint64_t) { if (c.rec < fail_rec) fail_rec = c.rec; }
};

// field lengths of the kept records into lens[col * (kept + 1) + rec]; the first failure key inside record fail_rec
struct LengthVisit {
    int64_t *lens;
    int64_t ncols, kept, fail_rec;
    uint64_t key = UINT64_MAX;
    LO_CSV_HD void keep(int64_t, const Carry &) {}
    LO_CSV_HD void save(const Carry &c) { if (c.rec < kept && c.col < ncols) lens[c.col * (kept + 1) + c.rec] = c.fbytes; }
    LO_CSV_HD void end(const Carry &) {}
    LO_CSV_HD void fail(const Carry &c, uint64_t k) { if (c.rec == fail_rec && k < key) key = k; }
};

// the kept bytes of the kept records to chars[offsets[col * (kept + 1) + rec] + offset in field]
struct ScatterVisit {
    const uint8_t *body;
    const int64_t *offsets;
    uint8_t *chars;
    int64_t ncols, kept;
    LO_CSV_HD void keep(int64_t p, const Carry &c) {
        if (c.rec < kept && c.col < ncols) chars[offsets[c.col * (kept + 1) + c.rec] + c.fbytes] = body[p];
    }
    LO_CSV_HD void save(const Carry &) {}
    LO_CSV_HD void end(const Carry &) {}
    LO_CSV_HD void fail(const Carry &, uint64_t) {}
};

// ---- a body fed in pieces: windows ----------------------------------------------------------------------------------
// Every record ends at a line end or at EOF, and the state after a record end is START_RECORD, so a body can be cut
// one past any byte that ended a record and the rest read as a body of its own.  Then the bytes before the cut are a
// complete body to the passes above: the EOF step does nothing there (the last byte is a line break, the state
// START_RECORD) and UTF-8 look-ahead meets that break before the cut.  The rest starts with a line break only when a
// run of breaks straddles the cut; it is then classed as a line end instead of skipped, which in START_RECORD is the
// same step.  What the later part needs from the earlier: the header's field count, and how many records and bytes
// came before it (record indices and failure positions are absolute in the whole body).

// Position in [b, e) of the last byte that ended a record, walking from state s; -1 if none.
LO_CSV_HD int64_t segment_last_end(const uint8_t *body, int64_t b, int64_t e, uint32_t s) {
    int64_t last = -1;
    int32_t prev = b > 0 ? (int32_t)body[b - 1] : -1;
    for (int64_t p = b; p < e; ++p) {
        const uint32_t t = step(s, byte_class(body[p], prev));
        prev = body[p];
        s = t & 7u;
        if ((t >> 4) & kEnd) last = p;
    }
    return last;
}

// The bookkeeping of a window [tail of the previous window | new bytes] of at most cap bytes.  A piece is taken into
// the window as far as it fits; a full window (or the body's last byte) is read up to its cut: one past the last byte
// that ended a record, or its whole length at the end of the body.  A full window in which no record ends doubles
// instead.  [cut, len) is the next window's tail.
struct StreamWindow {
    int64_t cap;             // bytes the window holds
    int64_t len = 0;         // bytes in it
    int64_t base = 0;        // offset of its first byte in the body
    int64_t rec0 = 0;        // records before it (absolute index of its first record)
    int64_t ncols = -1;      // the header's fields once record 0 has been read; -1 before
    LO_CSV_HD int64_t take(int64_t n) const { return n < cap - len ? n : cap - len; }
    LO_CSV_HD bool ready(bool final) const { return final || len == cap; }
    // last_end: the window's last byte that ended a record (-1: none); 0 -> grow the window
    LO_CSV_HD int64_t cut(int64_t last_end, bool final) const { return final ? len : last_end + 1; }
    LO_CSV_HD void grow() { cap *= 2; }
    // the window was read up to cut; nrec records ended in it, the first of them the header when rec0 == 0
    LO_CSV_HD void advance(int64_t cut, int64_t nrec, int64_t header_cols) {
        if (rec0 == 0 && nrec > 0) ncols = header_cols;
        base += cut;
        len -= cut;
        rec0 += nrec;
    }
};

}  // namespace csv
}  // namespace lo
