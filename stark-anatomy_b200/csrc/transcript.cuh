// transcript.cuh -- a proof's transcript read from its pickled bytes (DESIGN section 3.17): the grammar of the
// canonical pickle of a proof stream of one verifier plan's shape, the Fiat-Shamir messages the stream's
// verifier_fiat_shamir hashes (code/ip.py:24-25, code/fast_rpsss.py:16-17), SHAKE-256, blake2b over messages of any
// length, the draws of the weights, alphas and indices (fast_stark.py:73-74, algebra.py:116-120, fri.py:30-51) and
// the writers of the sections VerifierPlan._pack lays out.  __host__ __device__ so tests/emu runs the same code.
//
// The bytes come from outside the program: every read is checked against the proof's length and the current frame,
// every memo index against the memo entries made so far, every write stays inside the proof's own workspace.  A proof
// the grammar does not take is refused (its flag 0), and the caller verifies it on the host as before.
#pragma once
#include "../../include/sa_b200.h"
#include "hash.cuh"
#include "sample.cuh"

namespace sa {

// ---- the plan's shape: sa_transcript_* take it as SA_TRANSCRIPT_SHAPE 64-bit words ------------------------------
enum { TS_NREGS, TS_ROUNDS, TS_K, TS_LAST_LEN, TS_LOG_N, TS_NOPEN, TS_NWEIGHTS, TS_PROTO, TS_EF, TS_MEMO_CAP };

struct TShape {
    uint32_t nregs, rounds, k, last_len, log_n, nopen, nweights, proto, ef;
    uint64_t memo_cap;
    // objects of the stream, roots in front of everything, and the Fiat-Shamir messages (rounds + 2)
    SA_HD uint32_t nroots() const { return nregs + 1 + rounds; }
    SA_HD uint64_t nobjects() const { return (uint64_t)nroots() + 1 + (uint64_t)(rounds - 1) * 4 * k + 8ULL * nopen * k; }
    SA_HD uint32_t nfs() const { return rounds + 2; }
    // objects before Fiat-Shamir message m: the roots for the weights, one more FRI root per alpha, then the last
    // codeword for the indices
    SA_HD uint32_t fs_objects(uint32_t m) const { return m == 0 ? nregs + 1 : (m <= rounds ? nregs + 1 + m : nroots() + 1); }
    // digests in parse order: the roots, then per FRI round 3k paths (depths d, d, d - 1 with d = log_n - r), then
    // per opened codeword 4k paths of depth log_n
    SA_HD uint64_t fri_digests() const {
        uint64_t t = 0;
        for (uint32_t r = 0; r + 1 < rounds; r++) t += (uint64_t)k * (3 * (log_n - r) - 1);
        return t;
    }
    SA_HD uint64_t path_digests() const { return fri_digests() + 4ULL * nopen * k * log_n; }
    SA_HD uint64_t ndigests() const { return nroots() + path_digests(); }
    // elements in parse order: the last codeword, the triples of every round, the opened leaves
    SA_HD uint64_t nvalues() const { return last_len + 3ULL * (rounds - 1) * k + 4ULL * nopen * k; }
    SA_HD uint64_t npaths() const { return 3ULL * (rounds - 1) * k + 4ULL * nopen * k; }
    SA_HD uint64_t ncolinear() const { return (uint64_t)(rounds - 1) * k; }
};

// memo entries a canonical stream of the shape makes when no object is shared: the list of objects, every digest,
// every list, tuple, element and element dict, and the ten of the first element's class, strings and field
SA_HD uint64_t transcript_memo_cap(const TShape &s) {
    const uint64_t lists = 1 + 1 + 3ULL * (s.rounds - 1) * s.k + 4ULL * s.nopen * s.k;
    const uint64_t tuples = (uint64_t)(s.rounds - 1) * s.k;
    return lists + tuples + s.ndigests() + 2 * s.nvalues() + 10;
}

inline TShape transcript_shape(const uint64_t *w) {
    TShape s;
    s.nregs = (uint32_t)w[TS_NREGS];
    s.rounds = (uint32_t)w[TS_ROUNDS];
    s.k = (uint32_t)w[TS_K];
    s.last_len = (uint32_t)w[TS_LAST_LEN];
    s.log_n = (uint32_t)w[TS_LOG_N];
    s.nopen = (uint32_t)w[TS_NOPEN];
    s.nweights = (uint32_t)w[TS_NWEIGHTS];
    s.proto = (uint32_t)w[TS_PROTO];
    s.ef = (uint32_t)w[TS_EF];
    s.memo_cap = w[TS_MEMO_CAP];
    return s;
}

// the shapes sa_transcript_* take: a VerifierPlan's (1 to 16 registers, at least two FRI rounds, k distinct indices
// in the last codeword, a domain of 2^1 .. 2^30, the zerofier's codeword opened or not, every Fiat-Shamir prefix in
// the first batch of 1000 objects) with the memo capacity transcript_memo_cap gives
inline bool transcript_shape_ok(const uint64_t *w) {
    for (int i = 0; i < SA_TRANSCRIPT_SHAPE; i++)
        if (w[i] >= (1ULL << 32) && i != TS_MEMO_CAP) return false;
    const TShape s = transcript_shape(w);
    if (s.nregs < 1 || s.nregs > 16 || s.log_n < 1 || s.log_n > 30 || s.rounds < 2 || s.rounds > s.log_n) return false;
    if (s.last_len != (1u << (s.log_n - (s.rounds - 1))) || s.k < 1 || s.k > s.last_len) return false;
    if (s.nopen != s.nregs + 1 && s.nopen != s.nregs + 2) return false;
    if (s.nweights < 1 || s.nweights > 4096 || (s.proto != 4 && s.proto != 5) || s.ef >= (1u << s.log_n)) return false;
    if (s.nroots() + 1 > 1000) return false;
    return s.memo_cap == transcript_memo_cap(s);
}

// one proof's workspace: byte offsets of its sections, each 16-byte aligned
struct TLayout {
    uint64_t memo, kind, doff, vals, span, fsd, weights, alphas, top, status, total;
};
SA_HD uint64_t t_align(uint64_t x) { return (x + 15) & ~15ULL; }
SA_HD TLayout transcript_layout(const TShape &s) {
    TLayout l;
    uint64_t at = 0;
    l.memo = at; at += 16 * s.memo_cap;
    l.kind = at; at = t_align(at + s.memo_cap);
    l.doff = at; at = t_align(at + 8 * s.ndigests());
    l.vals = at; at += 16 * s.nvalues();
    l.span = at; at = t_align(at + 8 * (1 + s.nfs()));
    l.fsd = at; at += 32 * s.nfs();
    l.weights = at; at += 16 * (uint64_t)s.nweights;
    l.alphas = at; at += 16 * (uint64_t)s.rounds;
    l.top = at; at = t_align(at + 8 * (uint64_t)s.k);
    l.status = at; at += 16;
    l.total = at;
    return l;
}

// ---- the grammar ------------------------------------------------------------------------------------------------
enum : uint8_t {
    OP_MARK = 0x28, OP_STOP = 0x2e, OP_EMPTY_TUPLE = 0x29, OP_SHORT_BINBYTES = 0x43, OP_BININT = 0x4a,
    OP_BININT1 = 0x4b, OP_BININT2 = 0x4d, OP_APPEND = 0x61, OP_BUILD = 0x62, OP_APPENDS = 0x65, OP_BINGET = 0x68,
    OP_LONG_BINGET = 0x6a, OP_SETITEM = 0x73, OP_SETITEMS = 0x75, OP_EMPTY_LIST = 0x5d, OP_EMPTY_DICT = 0x7d,
    OP_PROTO = 0x80, OP_NEWOBJ = 0x81, OP_TUPLE3 = 0x87, OP_LONG1 = 0x8a, OP_SHORT_BINUNICODE = 0x8c,
    OP_STACK_GLOBAL = 0x93, OP_MEMOIZE = 0x94, OP_FRAME = 0x95
};
// what a memo entry holds; only digests, elements and the first element's class, strings and field may be named by
// a memo reference
enum : uint8_t {
    MK_OTHER, MK_DIGEST, MK_ELEM, MK_STR_MODULE, MK_STR_FE, MK_CLS_FE, MK_STR_VALUE, MK_STR_FIELD, MK_STR_FIELDCLS,
    MK_CLS_FIELD, MK_FIELD, MK_STR_P, MK_KINDS
};

#if defined(__CUDACC__)
#define SA_HD_CALL __host__ __device__ __noinline__
#else
#define SA_HD_CALL inline
#endif

struct TParser {
    const uint8_t *buf;
    uint64_t len, pos, frame_end, first_frame_end;
    fe *memo;
    uint8_t *kind;
    uint64_t memo_cap, nmemo;
    uint64_t have[MK_KINDS];  // memo index + 1 of the entry of each named kind, 0 before it is made
    uint64_t *doff;
    fe *vals;
    uint64_t ndig, nval, ndig_cap, nval_cap;
    bool framed;

    // the next opcode's byte, opening the next frame where the current one ends; -1 past the end or on a bad frame
    SA_HD int peek() {
        if (pos == frame_end) {
            if (pos >= len) return -1;
            if (buf[pos] == OP_FRAME) {
                if (len - pos < 9) return -1;
                uint64_t n = 0;
                for (int i = 7; i >= 0; i--) n = (n << 8) | buf[pos + 1 + i];
                if (n < 4 || n > len - pos - 9) return -1;
                pos += 9;
                frame_end = pos + n;
                if (!framed) first_frame_end = frame_end;
                framed = true;
            } else if (framed && len - pos < 4) {
                frame_end = len;  // the pickler writes a last frame of under four bytes unframed
            } else {
                return -1;
            }
        }
        return pos < frame_end ? buf[pos] : -1;
    }
    SA_HD bool op(uint8_t want) {
        if (peek() != want) return false;
        pos++;
        return true;
    }
    // n argument bytes of the opcode just read, inside the current frame
    SA_HD bool take(uint64_t n, uint64_t &at) {
        if (frame_end - pos < n) return false;
        at = pos;
        pos += n;
        return true;
    }
    SA_HD bool memoize(uint8_t k, fe v) {
        if (!op(OP_MEMOIZE) || nmemo >= memo_cap) return false;
        memo[nmemo] = v;
        kind[nmemo] = k;
        if (k != MK_OTHER && k != MK_DIGEST && k != MK_ELEM) have[k] = nmemo + 1;
        nmemo++;
        return true;
    }
    SA_HD bool is_get() {
        const int c = peek();
        return c == OP_BINGET || c == OP_LONG_BINGET;
    }
    // a memo reference: BINGET below 256, LONG_BINGET from 256 on, to an entry made so far of kind k
    SA_HD bool get(uint8_t k, uint64_t &idx) {
        uint64_t at;
        if (op(OP_BINGET)) {
            if (!take(1, at)) return false;
            idx = buf[at];
        } else if (op(OP_LONG_BINGET)) {
            if (!take(4, at)) return false;
            idx = (uint64_t)buf[at] | (uint64_t)buf[at + 1] << 8 | (uint64_t)buf[at + 2] << 16 |
                  (uint64_t)buf[at + 3] << 24;
            if (idx < 256) return false;
        } else {
            return false;
        }
        return idx < nmemo && kind[idx] == k;
    }
    // a string the pickler memoizes: a reference once it is in the memo, else written out in full
    SA_HD bool str(uint8_t k, const char *s, uint32_t n) {
        uint64_t idx, at;
        if (have[k]) return get(k, idx) && idx + 1 == have[k];
        if (!op(OP_SHORT_BINUNICODE) || !take(1, at) || buf[at] != n || !take(n, at)) return false;
        for (uint32_t i = 0; i < n; i++)
            if (buf[at + i] != (uint8_t)s[i]) return false;
        return memoize(k, fe_zero());
    }
    // STACK_GLOBAL('algebra', name): a reference once the class is in the memo
    SA_HD bool cls(uint8_t k, uint8_t name_kind, const char *name, uint32_t n) {
        uint64_t idx;
        if (have[k]) return get(k, idx);
        return str(MK_STR_MODULE, "algebra", 7) && str(name_kind, name, n) && op(OP_STACK_GLOBAL) &&
               memoize(k, fe_zero());
    }
    // a non-negative int as the pickler writes it: BININT1 below 2^8, BININT2 below 2^16, BININT below 2^31, else
    // LONG1 of bit_length / 8 + 1 bytes; at most 2^128 - 1 here
    SA_HD_CALL bool integer(fe &v) {
        uint64_t at;
        uint8_t b[16] = {0};
        uint32_t n;
        if (op(OP_BININT1)) {
            if (!take(1, at)) return false;
            n = 1;
        } else if (op(OP_BININT2)) {
            if (!take(2, at)) return false;
            n = 2;
            if (buf[at + 1] == 0) return false;
        } else if (op(OP_BININT)) {
            if (!take(4, at)) return false;
            n = 4;
            if ((buf[at + 3] == 0 && buf[at + 2] == 0) || (buf[at + 3] & 0x80)) return false;
        } else if (op(OP_LONG1)) {
            if (!take(1, at)) return false;
            n = buf[at];
            if (n < 5 || n > 17 || !take(n, at)) return false;
            // minimal: the top byte is a zero sign byte only when the next one has its top bit set, else the top
            // byte is non-zero with a clear top bit; and the value is not one BININT writes
            const uint8_t top = buf[at + n - 1], next = buf[at + n - 2];
            if (top & 0x80) return false;
            if (top == 0 && !(next & 0x80)) return false;
            if (n == 5 && top == 0 && next < 0x80) return false;
            if (n == 17) {
                if (top != 0) return false;
                n = 16;
            }
        } else {
            return false;
        }
        for (uint32_t i = 0; i < n; i++) b[i] = buf[at + i];
        v = fe_make(b[0] | b[1] << 8 | b[2] << 16 | (uint32_t)b[3] << 24, b[4] | b[5] << 8 | b[6] << 16 | (uint32_t)b[7] << 24,
                    b[8] | b[9] << 8 | b[10] << 16 | (uint32_t)b[11] << 24,
                    b[12] | b[13] << 8 | b[14] << 16 | (uint32_t)b[15] << 24);
        return true;
    }
    // the element's Field: a reference to the one Field, or (the first time) algebra.Field() with {'p': p}
    SA_HD bool field() {
        uint64_t idx;
        if (have[MK_FIELD]) return get(MK_FIELD, idx);
        fe p;
        if (!cls(MK_CLS_FIELD, MK_STR_FIELDCLS, "Field", 5) || !op(OP_EMPTY_TUPLE) || !op(OP_NEWOBJ)) return false;
        const uint64_t self = nmemo;
        if (!memoize(MK_OTHER, fe_zero()) || !op(OP_EMPTY_DICT) || !memoize(MK_OTHER, fe_zero()) ||
            !str(MK_STR_P, "p", 1) || !integer(p) || !fe_eq(p, fe_make(1, 0, 0, P3)) || !op(OP_SETITEM) ||
            !op(OP_BUILD))
            return false;
        kind[self] = MK_FIELD;  // named only once its state is the field of p
        have[MK_FIELD] = self + 1;
        return true;
    }
    SA_HD_CALL bool element(fe &v) {
        uint64_t idx;
        // a reference names an earlier element, or else the class that starts a new element's encoding
        const uint64_t at = pos, fend = frame_end, first = first_frame_end;
        const bool was_framed = framed;
        if (is_get() && get(MK_ELEM, idx)) {
            v = memo[idx];
            return true;
        }
        pos = at;
        frame_end = fend;
        first_frame_end = first;
        framed = was_framed;
        if (!cls(MK_CLS_FE, MK_STR_FE, "FieldElement", 12) || !op(OP_EMPTY_TUPLE) || !op(OP_NEWOBJ)) return false;
        const uint64_t self = nmemo;
        if (!memoize(MK_OTHER, fe_zero()) || !op(OP_EMPTY_DICT) || !memoize(MK_OTHER, fe_zero()) || !op(OP_MARK) ||
            !str(MK_STR_VALUE, "value", 5) || !integer(v) || !str(MK_STR_FIELD, "field", 5) || !field() ||
            !op(OP_SETITEMS) || !op(OP_BUILD))
            return false;
        const fe p = fe_make(1, 0, 0, P3);
        for (int i = 3; i >= 0; i--) {  // a value at or above p is refused
            if (v.v[i] < p.v[i]) break;
            if (v.v[i] > p.v[i] || i == 0) return false;
        }
        memo[self] = v;
        kind[self] = MK_ELEM;  // a reference inside its own state would have named an unfinished element
        return true;
    }
    SA_HD bool value() {
        fe v;
        if (nval >= nval_cap || !element(v)) return false;
        vals[nval++] = v;
        return true;
    }
    SA_HD_CALL bool digest() {
        uint64_t at;
        if (ndig >= ndig_cap) return false;
        if (is_get()) {
            uint64_t idx;
            if (!get(MK_DIGEST, idx)) return false;
            doff[ndig++] = ((uint64_t)memo[idx].v[1] << 32) | memo[idx].v[0];
            return true;
        }
        if (!op(OP_SHORT_BINBYTES) || !take(1, at) || buf[at] != 64 || !take(64, at)) return false;
        doff[ndig++] = at;
        return memoize(MK_DIGEST, fe_from_u64(at));
    }
    // a list of n items: EMPTY_LIST MEMOIZE, then APPEND for one item, else MARK ... APPENDS per batch of 1000
    template <typename F>
    SA_HD bool list(uint64_t n, F &&item) {
        if (!op(OP_EMPTY_LIST) || !memoize(MK_OTHER, fe_zero())) return false;
        if (n == 1) return item(0) && op(OP_APPEND);
        for (uint64_t done = 0; done < n;) {
            if (!op(OP_MARK)) return false;
            for (uint64_t b = 0; b < 1000 && done < n; b++, done++)
                if (!item(done)) return false;
            if (!op(OP_APPENDS)) return false;
        }
        return true;
    }
    SA_HD bool path(uint32_t depth);
    SA_HD bool triple() {
        return value() && value() && value() && op(OP_TUPLE3) && memoize(MK_OTHER, fe_zero());
    }
};

struct TDigest {
    TParser *p;
    SA_HD bool operator()(uint64_t) { return p->digest(); }
};
struct TValue {
    TParser *p;
    SA_HD bool operator()(uint64_t) { return p->value(); }
};
SA_HD bool TParser::path(uint32_t depth) { return list(depth, TDigest{this}); }

// the stream's objects in order, object t at each call: the roots, the last codeword, per FRI round k triples and
// 3k paths of depths d, d, d - 1 (d = log_n - r), then per opened codeword 4k (leaf, path) pairs; the Fiat-Shamir
// spans recorded on the way
struct TObjects {
    TParser *p;
    const TShape *s;
    uint64_t *span;
    uint64_t t;
    uint32_t r, q, o;  // the round, object within a round and opened codeword of the next object
    SA_HD bool operator()(uint64_t) {
        bool ok;
        const uint32_t nroots = s->nroots();
        if (t == 0) span[0] = p->pos;
        if (t < nroots) {
            ok = p->digest();
        } else if (t == nroots) {
            ok = p->list(s->last_len, TValue{p});
        } else if (r + 1 < s->rounds) {
            ok = q < s->k ? p->triple() : p->path(s->log_n - r - ((q - s->k) % 3 == 2));
            if (++q == 4 * s->k) q = 0, r++;
        } else {
            ok = (q & 1) ? p->path(s->log_n) : p->value();
            if (++q == 8 * s->k) q = 0, o++;
        }
        t++;
        for (uint32_t m = 0; m < s->nfs(); m++)
            if (t == s->fs_objects(m)) span[1 + m] = p->pos;
        return ok;
    }
};

// Parse one proof.  On acceptance: doff[] holds the byte offset in the proof of every digest in parse order,
// vals[] every element's canonical value in parse order, and span[0] the offset of the first object, span[1 + m]
// the end of the last object of Fiat-Shamir message m.  Returns the accepted flag.
SA_HD bool transcript_parse(const uint8_t *buf, uint64_t len, const TShape &s, uint8_t *ws, const TLayout &l) {
    TParser p;
    p.buf = buf;
    p.len = len;
    p.pos = 0;
    p.frame_end = 2;  // PROTO is written before the first frame
    p.first_frame_end = 0;
    p.memo = (fe *)(ws + l.memo);
    p.kind = ws + l.kind;
    p.memo_cap = s.memo_cap;
    p.nmemo = 0;
    for (int i = 0; i < MK_KINDS; i++) p.have[i] = 0;
    p.doff = (uint64_t *)(ws + l.doff);
    p.vals = (fe *)(ws + l.vals);
    p.ndig = p.nval = 0;
    p.ndig_cap = s.ndigests();
    p.nval_cap = s.nvalues();
    p.framed = false;
    uint64_t *span = (uint64_t *)(ws + l.span);
    if (len < 2 || buf[0] != OP_PROTO || buf[1] != s.proto) return false;
    p.pos = 2;
    TObjects object{&p, &s, span, 0, 0, 0, 0};
    if (!p.list(s.nobjects(), object) || !p.op(OP_STOP) || p.pos != len || p.frame_end != len) return false;
    if (!p.framed || p.ndig != p.ndig_cap || p.nval != p.nval_cap || object.o != s.nopen) return false;
    // every Fiat-Shamir prefix lies in the first frame, and its own pickle fits one frame
    for (uint32_t m = 0; m < s.nfs(); m++)
        if (span[1 + m] > p.first_frame_end || span[1 + m] - span[0] + 5 >= 65536) return false;
    return true;
}

// ---- SHAKE-256 -----------------------------------------------------------------------------------------------------
SA_HD uint64_t k_rotl(uint64_t x, int r) { return r ? (x << r) | (x >> (64 - r)) : x; }

SA_HD void keccak_f1600(uint64_t a[25]) {
    const uint64_t rc[24] = {0x0000000000000001ULL, 0x0000000000008082ULL, 0x800000000000808aULL,
                             0x8000000080008000ULL, 0x000000000000808bULL, 0x0000000080000001ULL,
                             0x8000000080008081ULL, 0x8000000000008009ULL, 0x000000000000008aULL,
                             0x0000000000000088ULL, 0x0000000080008009ULL, 0x000000008000000aULL,
                             0x000000008000808bULL, 0x800000000000008bULL, 0x8000000000008089ULL,
                             0x8000000000008003ULL, 0x8000000000008002ULL, 0x8000000000000080ULL,
                             0x000000000000800aULL, 0x800000008000000aULL, 0x8000000080008081ULL,
                             0x8000000000008080ULL, 0x0000000080000001ULL, 0x8000000080008008ULL};
    // rho offsets and pi's destination along the lane walk (1, 0) -> ...
    const int rho[24] = {1, 3, 6, 10, 15, 21, 28, 36, 45, 55, 2, 14, 27, 41, 56, 8, 25, 43, 62, 18, 39, 61, 20, 44};
    const int pi[24] = {10, 7, 11, 17, 18, 3, 5, 16, 8, 21, 24, 4, 15, 23, 19, 13, 12, 2, 20, 14, 22, 9, 6, 1};
    for (int round = 0; round < 24; round++) {
        uint64_t c[5];
        for (int x = 0; x < 5; x++) c[x] = a[x] ^ a[x + 5] ^ a[x + 10] ^ a[x + 15] ^ a[x + 20];
        for (int x = 0; x < 5; x++) {
            const uint64_t d = c[(x + 4) % 5] ^ k_rotl(c[(x + 1) % 5], 1);
            for (int y = 0; y < 25; y += 5) a[y + x] ^= d;
        }
        uint64_t cur = a[1];
        for (int i = 0; i < 24; i++) {
            const int j = pi[i];
            const uint64_t tmp = a[j];
            a[j] = k_rotl(cur, rho[i]);
            cur = tmp;
        }
        for (int y = 0; y < 25; y += 5) {
            const uint64_t b0 = a[y], b1 = a[y + 1], b2 = a[y + 2], b3 = a[y + 3], b4 = a[y + 4];
            a[y] = b0 ^ (~b1 & b2);
            a[y + 1] = b1 ^ (~b2 & b3);
            a[y + 2] = b2 ^ (~b3 & b4);
            a[y + 3] = b3 ^ (~b4 & b0);
            a[y + 4] = b4 ^ (~b0 & b1);
        }
        a[0] ^= rc[round];
    }
}

// SHAKE-256 absorbing byte by byte (rate 136)
struct Shake256 {
    uint64_t a[25];
    uint32_t at;
    SA_HD void init() {
        for (int i = 0; i < 25; i++) a[i] = 0;
        at = 0;
    }
    SA_HD void byte(uint8_t b) {
        a[at >> 3] ^= (uint64_t)b << (8 * (at & 7));
        if (++at == 136) {
            keccak_f1600(a);
            at = 0;
        }
    }
    SA_HD void bytes(const uint8_t *p, uint64_t n) {
        for (uint64_t i = 0; i < n; i++) byte(p[i]);
    }
    // the first 32 bytes of the output: lanes 0..3, little-endian
    SA_HD void final32(uint64_t out[4]) {
        a[at >> 3] ^= 0x1FULL << (8 * (at & 7));
        a[135 >> 3] ^= 0x80ULL << (8 * (135 & 7));
        keccak_f1600(a);
        for (int i = 0; i < 4; i++) out[i] = a[i];
    }
};

// shake_256(prefix + pickle.dumps(objects[:j])).digest(32) from the proof's own bytes of those j objects: PROTO,
// FRAME with the prefix's frame length, EMPTY_LIST MEMOIZE (MARK for j >= 2), the objects, then APPENDS STOP
// (APPEND STOP for j = 1)
SA_HD void transcript_fs_digest(uint64_t out[4], const uint8_t *prefix, uint32_t nprefix, uint32_t proto,
                                const uint8_t *body, uint64_t nbody, uint32_t j) {
    Shake256 h;
    h.init();
    h.bytes(prefix, nprefix);
    const uint64_t frame = (j >= 2 ? 3 : 2) + nbody + 2;
    h.byte(OP_PROTO);
    h.byte((uint8_t)proto);
    h.byte(OP_FRAME);
    for (int i = 0; i < 8; i++) h.byte((uint8_t)(frame >> (8 * i)));
    h.byte(OP_EMPTY_LIST);
    h.byte(OP_MEMOIZE);
    if (j >= 2) h.byte(OP_MARK);
    h.bytes(body, nbody);
    h.byte(j >= 2 ? OP_APPENDS : OP_APPEND);
    h.byte(OP_STOP);
    h.final32(out);
}

// ---- blake2b of seed (32 bytes) || `zeros` zero bytes, the message hashlib.blake2b(seed + bytes(zeros)) hashes ----
SA_HD void blake2b_compress(uint64_t h[8], const uint64_t m[16], uint64_t t, bool last) {
    const uint64_t iv0 = 0x6a09e667f3bcc908ULL, iv1 = 0xbb67ae8584caa73bULL, iv2 = 0x3c6ef372fe94f82bULL,
                   iv3 = 0xa54ff53a5f1d36f1ULL, iv4 = 0x510e527fade682d1ULL, iv5 = 0x9b05688c2b3e6c1fULL,
                   iv6 = 0x1f83d9abfb41bd6bULL, iv7 = 0x5be0cd19137e2179ULL;
    uint64_t v0 = h[0], v1 = h[1], v2 = h[2], v3 = h[3], v4 = h[4], v5 = h[5], v6 = h[6], v7 = h[7];
    uint64_t v8 = iv0, v9 = iv1, v10 = iv2, v11 = iv3, v12 = iv4 ^ t, v13 = iv5, v14 = last ? ~iv6 : iv6,
             v15 = iv7;
    SA_B2_ROUND(0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15);
    SA_B2_ROUND(14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3);
    SA_B2_ROUND(11, 8, 12, 0, 5, 2, 15, 13, 10, 14, 3, 6, 7, 1, 9, 4);
    SA_B2_ROUND(7, 9, 3, 1, 13, 12, 11, 14, 2, 6, 5, 10, 4, 0, 15, 8);
    SA_B2_ROUND(9, 0, 5, 7, 2, 4, 10, 15, 14, 1, 11, 12, 6, 8, 3, 13);
    SA_B2_ROUND(2, 12, 6, 10, 0, 11, 8, 3, 4, 13, 7, 5, 15, 14, 1, 9);
    SA_B2_ROUND(12, 5, 1, 15, 14, 13, 4, 10, 0, 7, 6, 3, 9, 2, 8, 11);
    SA_B2_ROUND(13, 11, 7, 14, 12, 1, 3, 9, 5, 0, 15, 4, 8, 6, 2, 10);
    SA_B2_ROUND(6, 15, 14, 9, 11, 3, 0, 8, 12, 2, 13, 7, 1, 4, 10, 5);
    SA_B2_ROUND(10, 2, 8, 4, 7, 6, 1, 5, 15, 11, 9, 14, 3, 12, 13, 0);
    SA_B2_ROUND(0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15);
    SA_B2_ROUND(14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3);
    h[0] ^= v0 ^ v8;
    h[1] ^= v1 ^ v9;
    h[2] ^= v2 ^ v10;
    h[3] ^= v3 ^ v11;
    h[4] ^= v4 ^ v12;
    h[5] ^= v5 ^ v13;
    h[6] ^= v6 ^ v14;
    h[7] ^= v7 ^ v15;
}

SA_HD void blake2b_seed_zeros(uint64_t out[8], const uint64_t seed[4], uint64_t zeros) {
    out[0] = 0x6a09e667f3bcc908ULL ^ 0x01010040ULL;
    out[1] = 0xbb67ae8584caa73bULL;
    out[2] = 0x3c6ef372fe94f82bULL;
    out[3] = 0xa54ff53a5f1d36f1ULL;
    out[4] = 0x510e527fade682d1ULL;
    out[5] = 0x9b05688c2b3e6c1fULL;
    out[6] = 0x1f83d9abfb41bd6bULL;
    out[7] = 0x5be0cd19137e2179ULL;
    const uint64_t total = 32 + zeros;
    uint64_t m[16];
    for (int i = 0; i < 16; i++) m[i] = i < 4 ? seed[i] : 0;
    // every block but the last is full; the last holds the remaining 1..128 bytes
    uint64_t done = 0;
    while (total - done > 128) {
        done += 128;
        blake2b_compress(out, m, done, false);
        for (int i = 0; i < 4; i++) m[i] = 0;
    }
    blake2b_compress(out, m, total, true);
}

// ---- big-endian integers mod p (Field.sample) --------------------------------------------------------------------
// 16 big-endian bytes of a little-endian word stream starting at byte `at`, reduced below p (2^128 < 2p)
SA_HD fe t_limb_be(const uint64_t *w, int at) {
    uint32_t x[4];
    for (int i = 0; i < 4; i++) {
        uint32_t v = 0;
        for (int b = 0; b < 4; b++) {
            const int k = at + 4 * (3 - i) + b;  // limb i (least significant first) is bytes 12 - 4i .. 15 - 4i
            v = (v << 8) | (uint32_t)((w[k >> 3] >> (8 * (k & 7))) & 0xFF);
        }
        x[i] = v;
    }
    const fe p = fe_make(1, 0, 0, P3);
    bool ge = true;
    for (int i = 3; i >= 0; i--)
        if (x[i] != p.v[i]) {
            ge = x[i] > p.v[i];
            break;
        }
    const fe v = fe_make(x[0], x[1], x[2], x[3]);
    return ge ? fe_sub(v, p) : v;
}
// int.from_bytes(bytes(32 * nwords ... )) mod p for the nbytes (a multiple of 16) of a digest's words
SA_HD fe transcript_reduce_be(const uint64_t *w, int nbytes) {
    const fe r = fe_mont_one();  // 2^128 mod p, in normal form; fe_mul(a, b) = a b mod p for normal a and b
    fe acc = t_limb_be(w, 0);
    for (int at = 16; at < nbytes; at += 16) acc = fe_add(fe_mul(acc, r), t_limb_be(w, at));
    return acc;
}

// index draws stop after this many counters over the needed k; the host verifies such a proof
SA_HD uint64_t transcript_counter_cap(const TShape &s) { return 64ULL * s.last_len + 4096; }

// the weights, alphas and indices of one accepted proof from its Fiat-Shamir digests; false when the index loop
// passes transcript_counter_cap
SA_HD bool transcript_draws(const TShape &s, uint8_t *ws, const TLayout &l) {
    const uint64_t *fsd = (const uint64_t *)(ws + l.fsd);
    fe *weights = (fe *)(ws + l.weights), *alphas = (fe *)(ws + l.alphas);
    uint64_t *top = (uint64_t *)(ws + l.top);
    uint64_t d[8];
    for (uint32_t i = 0; i < s.nweights; i++) {
        blake2b_seed_zeros(d, fsd, i);
        weights[i] = transcript_reduce_be(d, 64);
    }
    for (uint32_t r = 0; r < s.rounds; r++) alphas[r] = transcript_reduce_be(fsd + 4 * (1 + r), 32);
    const uint64_t size = 1ULL << (s.log_n - 1), cap = transcript_counter_cap(s);
    uint32_t found = 0;
    for (uint64_t counter = 0; found < s.k; counter++) {
        if (counter >= cap) return false;
        blake2b_seed_zeros(d, fsd + 4 * (1 + s.rounds), counter);
        const uint64_t index = sample_bswap64(d[7]) & (size - 1);  // the big-endian value mod a power of two
        bool fresh = true;
        for (uint32_t i = 0; i < found; i++)
            if (((top[i] ^ index) & (s.last_len - 1)) == 0) fresh = false;
        if (fresh) top[found++] = index;
    }
    return true;
}

// ---- the sections of VerifierPlan._pack ---------------------------------------------------------------------------
// section byte offsets, SA_TRANSCRIPT_SECTIONS of them, in _pack's order
enum {
    SEC_ROOTS, SEC_LEAVES, SEC_LEAF_INDEX, SEC_DEPTH, SEC_DIGESTS, SEC_PATH_OFFSET, SEC_AY, SEC_BY, SEC_CY, SEC_ALPHA,
    SEC_ITEMS, SEC_PROOF_DATA, SEC_LAST, SEC_A_INDEX, SEC_ROUND
};

SA_HD void t_copy64(uint8_t *dst, const uint8_t *src, bool ok) {
    for (int i = 0; i < 64; i++) dst[i] = ok ? src[i] : 0;
}

// the first of the 2k combination values: entry e < k is round 0's a-value at top[e] mod n/2, entry k + e its
// b-value at that index + n/2
SA_HD uint64_t t_entry_index(const uint64_t *top, uint32_t k, uint64_t half, uint32_t e) {
    return e < k ? top[e] & (half - 1) : (top[e - k] & (half - 1)) + half;
}
// the 4k opened indices in pull order before sorting: the 2k entry indices, then each + ef mod n
SA_HD uint64_t t_dup_value(const uint64_t *top, const TShape &s, uint32_t u) {
    const uint64_t n = 1ULL << s.log_n;
    return u < 2 * s.k ? t_entry_index(top, s.k, n >> 1, u) : (t_entry_index(top, s.k, n >> 1, u - 2 * s.k) + s.ef) & (n - 1);
}
// the position in the sorted opened indices of the last read of index x (a repeated index keeps the last leaf)
SA_HD uint32_t t_last_position(const uint64_t *top, const TShape &s, uint64_t x) {
    uint32_t below = 0;
    for (uint32_t u = 0; u < 4 * s.k; u++) below += t_dup_value(top, s, u) <= x;
    return below - 1;
}

// path q of proof b: its root, leaf, depth, path offset and (for FRI paths) leaf index
SA_HD void transcript_path_elem(uint8_t *sec, const uint64_t *at, const TShape &s, const uint8_t *proof, uint8_t *ws,
                                const TLayout &l, const uint8_t *zroot, uint64_t b, uint64_t q) {
    const bool ok = *(const uint32_t *)(ws + l.status) != 0;
    const uint64_t *doff = (const uint64_t *)(ws + l.doff), *top = (const uint64_t *)(ws + l.top);
    const fe *vals = (const fe *)(ws + l.vals);
    const uint64_t gi = b * s.npaths() + q, nfri = 3ULL * (s.rounds - 1) * s.k;
    const uint8_t *root;
    fe leaf;
    uint32_t depth;
    uint64_t off = b * s.path_digests();
    if (q < nfri) {
        const uint32_t r = (uint32_t)(q / (3 * s.k)), w = (uint32_t)(q % (3 * s.k)), e = w / 3, c = w % 3;
        const uint32_t d = s.log_n - r;
        for (uint32_t i = 0; i < r; i++) off += (uint64_t)s.k * (3 * (s.log_n - i) - 1);
        off += (uint64_t)e * (3 * d - 1) + (c >= 1 ? d : 0) + (c == 2 ? d : 0);
        root = proof + (ok ? doff[s.nregs + 1 + r + (c == 2)] : 0);
        leaf = vals[s.last_len + 3ULL * (r * s.k + e) + c];
        depth = d - (c == 2);
        const uint64_t half = 1ULL << (s.log_n - r - 1);
        const uint64_t a = ok ? top[e] & (half - 1) : 0;
        ((uint64_t *)(sec + at[SEC_LEAF_INDEX]))[gi] = c == 1 ? a + half : a;
    } else {
        const uint64_t j = q - nfri, o = j / (4 * s.k);
        off += s.fri_digests() + j * s.log_n;
        root = o < s.nregs + 1 ? proof + (ok ? doff[o] : 0) : zroot;
        leaf = vals[s.last_len + 3ULL * (s.rounds - 1) * s.k + j];
        depth = s.log_n;
    }
    t_copy64(sec + at[SEC_ROOTS] + 64 * gi, root, ok);
    ((fe *)(sec + at[SEC_LEAVES]))[gi] = ok ? leaf : fe_zero();
    ((uint32_t *)(sec + at[SEC_DEPTH]))[gi] = depth;
    ((uint64_t *)(sec + at[SEC_PATH_OFFSET]))[gi] = off;
}

// digest t of proof b's paths
SA_HD void transcript_digest_elem(uint8_t *sec, const uint64_t *at, const TShape &s, const uint8_t *proof,
                                  const uint8_t *ws, const TLayout &l, uint64_t b, uint64_t t) {
    const bool ok = *(const uint32_t *)(ws + l.status) != 0;
    const uint64_t *doff = (const uint64_t *)(ws + l.doff);
    t_copy64(sec + at[SEC_DIGESTS] + 64 * (b * s.path_digests() + t), ok ? proof + doff[s.nroots() + t] : proof, ok);
}

// everything else of proof b: the colinearity items, the opened leaves' indices, the combination items, proof_data
// (the weights, then the statement's `nstat` elements the host wrote) and the last codeword; and out (80 bytes: the
// accepted flag, then at 16 the last FRI root)
SA_HD void transcript_proof_elem(uint8_t *sec, const uint64_t *at, const TShape &s, const uint8_t *proof,
                                 uint8_t *ws, const TLayout &l, const fe *statement, uint64_t nstat, uint8_t *out,
                                 uint64_t b) {
    const bool ok = *(const uint32_t *)(ws + l.status) != 0;
    const uint64_t *doff = (const uint64_t *)(ws + l.doff), *top = (const uint64_t *)(ws + l.top);
    const fe *vals = (const fe *)(ws + l.vals), *weights = (const fe *)(ws + l.weights);
    const fe *alphas = (const fe *)(ws + l.alphas);
    const fe zero = fe_zero();
    const uint64_t ncol = s.ncolinear();
    for (uint32_t r = 0; r + 1 < s.rounds; r++) {
        const uint64_t half = 1ULL << (s.log_n - r - 1);
        for (uint32_t e = 0; e < s.k; e++) {
            const uint64_t i = b * ncol + (uint64_t)r * s.k + e;
            const fe *t = vals + s.last_len + 3ULL * (r * s.k + e);
            ((fe *)(sec + at[SEC_AY]))[i] = ok ? t[0] : zero;
            ((fe *)(sec + at[SEC_BY]))[i] = ok ? t[1] : zero;
            ((fe *)(sec + at[SEC_CY]))[i] = ok ? t[2] : zero;
            ((fe *)(sec + at[SEC_ALPHA]))[i] = ok ? alphas[r] : zero;
            ((uint64_t *)(sec + at[SEC_A_INDEX]))[i] = ok ? top[e] & (half - 1) : 0;
            ((uint32_t *)(sec + at[SEC_ROUND]))[i] = r;
        }
    }
    const uint32_t K = 4 * s.k;
    const uint64_t nfri = 3ULL * (s.rounds - 1) * s.k, open0 = s.last_len + 3ULL * (s.rounds - 1) * s.k;
    const uint64_t n = 1ULL << s.log_n;
    // opened index u goes to its sorted position (equal indices are equal values, so their order does not matter)
    for (uint32_t u = 0; u < K; u++) {
        const uint64_t x = ok ? t_dup_value(top, s, u) : 0;
        uint32_t pos = 0;
        for (uint32_t v = 0; v < K; v++) {
            const uint64_t y = ok ? t_dup_value(top, s, v) : 0;
            pos += y < x || (y == x && v < u);
        }
        for (uint32_t o = 0; o < s.nopen; o++)
            ((uint64_t *)(sec + at[SEC_LEAF_INDEX]))[b * s.npaths() + nfri + (uint64_t)o * K + pos] = x;
    }
    // the combination items in index order: [i, value, cur leaves, next leaves, the two extra codewords' leaves]
    const uint32_t R = 4 + 2 * s.nregs;
    fe *items = (fe *)(sec + at[SEC_ITEMS]);
    for (uint32_t e = 0; e < 2 * s.k; e++) {
        const uint64_t i = ok ? t_entry_index(top, s.k, n >> 1, e) : 0;
        uint32_t rank = 0;
        for (uint32_t f = 0; f < 2 * s.k; f++) rank += ok ? t_entry_index(top, s.k, n >> 1, f) < i : f < e;
        fe *it = items + (b * 2 * s.k + rank) * R;
        const uint32_t pi = ok ? t_last_position(top, s, i) : 0, pj = ok ? t_last_position(top, s, (i + s.ef) & (n - 1)) : 0;
        it[0] = fe_from_u64(i);
        it[1] = ok ? vals[s.last_len + 3ULL * (e % s.k) + (e >= s.k)] : zero;
        for (uint32_t g = 0; g < s.nregs; g++) {
            it[2 + g] = ok ? vals[open0 + (uint64_t)g * K + pi] : zero;
            it[2 + s.nregs + g] = ok ? vals[open0 + (uint64_t)g * K + pj] : zero;
        }
        it[2 + 2 * s.nregs] = ok ? vals[open0 + (uint64_t)s.nregs * K + pi] : zero;
        it[3 + 2 * s.nregs] = ok && s.nopen > s.nregs + 1 ? vals[open0 + (uint64_t)(s.nregs + 1) * K + pi] : zero;
    }
    fe *pdata = (fe *)(sec + at[SEC_PROOF_DATA]) + b * (s.nweights + nstat);
    for (uint32_t i = 0; i < s.nweights; i++) pdata[i] = ok ? weights[i] : zero;
    for (uint64_t i = 0; i < nstat; i++) pdata[s.nweights + i] = statement[b * nstat + i];
    fe *last = (fe *)(sec + at[SEC_LAST]) + b * s.last_len;
    for (uint32_t i = 0; i < s.last_len; i++) last[i] = ok ? vals[i] : zero;
    *(uint32_t *)out = ok;
    t_copy64(out + 16, proof + (ok ? doff[s.nroots() - 1] : 0), ok);
}

}  // namespace sa
