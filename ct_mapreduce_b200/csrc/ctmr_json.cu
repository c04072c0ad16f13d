// ctmr_json.cu -- kernels that find the entries of whole get-entries response bodies (ctmr_process_raw_bodies,
// include/ctmr_frontend.h) with Go 1.13 encoding/json's rules: Unmarshal of the body into ct.GetEntriesResponse after
// checkValid over all of it (reference cmd/ct-fetch/ct-fetch.go:424).
//
//   classify   one thread per 64-byte block of the staged bodies: masks of backslashes and quotes, the escaped
//              characters (odd backslash runs) and the in-string mask (prefix XOR of the unescaped quotes), simdjson's
//              stage 1.  Two carries cross a block edge: a backslash run that escapes the next block's first byte, and
//              the in-string parity.  A block's effect on them is a function of 2 bits -> 2 bits, so pass 1 writes each
//              block's function as a 4-entry table, a scan composes the tables, and pass 2 classifies each block with
//              its carries.  Both carries restart at every body start (bit arithmetic per segment of the block), which
//              also makes a block holding a body start a constant function: the scan needs no segment flags.
//   walk       one warp per body over the masks: every lane runs the same serial walk of the grammar (so the warp never
//              diverges) while the 32 lanes load 32 blocks of masks at a time to find the next token.  It validates the
//              grammar, checks scalars from the bytes and writes each entry's two spans into the body's slots.  The
//              warp reads the token mask directly; a compacted index of token positions would cost 4 bytes per token
//              and one more scan and would be read in the same order.
//   compact    per-body counts -> dense entry positions (a scan), spans and caller offsets to them.
//   unescape   one thread per string that held a backslash: the JSON escapes undone into the stage's spare half, '\r'
//              and '\n' dropped (base64.StdEncoding skips them), a non-ASCII character made one byte outside the
//              alphabet (the string is BAD_BASE64 either way).
#include <cub/device/device_scan.cuh>

#include "ctmr_common.cuh"

namespace ctmr {
namespace {

constexpr uint64_t kEven = 0x5555555555555555ull;
// byte classes (shared-memory table)
constexpr uint8_t C_BS = 1, C_QT = 2, C_ST = 4, C_WS = 8, C_CTL = 16, C_ESC = 32, C_U = 64, C_HEX = 128;

__device__ void fill_class_lut(uint8_t* lut) {
    for (uint32_t c = threadIdx.x; c < 256; c += blockDim.x) {
        uint8_t k = 0;
        if (c == '\\') k |= C_BS | C_ESC;
        if (c == '"') k |= C_QT | C_ESC;
        if (c == '{' || c == '}' || c == '[' || c == ']' || c == ':' || c == ',') k |= C_ST;
        if (c == ' ' || c == '\t' || c == '\n' || c == '\r') k |= C_WS;
        if (c < 0x20) k |= C_CTL;
        if (c == '/' || c == 'b' || c == 'f' || c == 'n' || c == 'r' || c == 't' || c == 'u') k |= C_ESC;
        if (c == 'u') k |= C_U;
        if ((c >= '0' && c <= '9') || (c >= 'a' && c <= 'f') || (c >= 'A' && c <= 'F')) k |= C_HEX;
        lut[c] = k;
    }
}

struct BlockBits {
    uint64_t bs = 0, qt = 0, st = 0, ws = 0, ctl = 0, esc = 0, u = 0;
};

__device__ __forceinline__ BlockBits load_block(const uint8_t* lut, const uint8_t* t, bool all) {
    BlockBits b;
    const uint4* v = reinterpret_cast<const uint4*>(t);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const uint4 w = v[q];
        const uint32_t words[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            const uint8_t k = lut[(words[i >> 2] >> (8 * (i & 3))) & 0xffu];
            const uint64_t bit = 1ull << (16 * q + i);
            b.bs |= (k & C_BS) ? bit : 0;
            b.qt |= (k & C_QT) ? bit : 0;
            if (all) {
                b.st |= (k & C_ST) ? bit : 0;
                b.ws |= (k & C_WS) ? bit : 0;
                b.ctl |= (k & C_CTL) ? bit : 0;
                b.esc |= (k & C_ESC) ? bit : 0;
                b.u |= (k & C_U) ? bit : 0;
            }
        }
    }
    return b;
}

__device__ __forceinline__ uint64_t prefix_xor(uint64_t x) {
    x ^= x << 1;
    x ^= x << 2;
    x ^= x << 4;
    x ^= x << 8;
    x ^= x << 16;
    x ^= x << 32;
    return x;
}

// One block: backslashes bs, quotes qt, body starts S, carry-in state (bit 0: the first byte is escaped, bit 1: inside a
// string).  Writes the escaped characters and the in-string mask (opening quote in, closing quote out); returns the
// carry-out state.  Segments [a, b) between body starts are done with simdjson's arithmetic shifted to bit 0.
__device__ __forceinline__ uint32_t scan_block(uint64_t bs, uint64_t qt, uint64_t S, uint32_t state, uint64_t* escd_out, uint64_t* instr_out) {
    uint32_t esc = state & 1u, str = state >> 1;
    uint64_t escd = 0, instr = 0;
    uint32_t a = 0;
    uint64_t rest = S;
    for (;;) {
        if ((rest >> a) & 1ull) {  // a body starts here: both carries restart
            esc = 0;
            str = 0;
            rest &= ~(1ull << a);
        }
        const uint32_t b = rest ? (uint32_t)(__ffsll((long long)rest) - 1) : 64u;
        const uint32_t L = b - a;
        const uint64_t seg = L == 64 ? ~0ull : ((1ull << L) - 1);
        const uint64_t B = (bs >> a) & seg & ~(uint64_t)esc;  // an escaped first byte escapes nothing itself
        const uint64_t follows = (B << 1) | (uint64_t)esc;
        const uint64_t odd_starts = B & ~kEven & ~follows;
        const uint64_t sum = odd_starts + B;
        uint64_t e = (kEven ^ (sum << 1)) & follows;
        const uint32_t esc_next = L == 64 ? (uint32_t)(sum < B) : (uint32_t)((e >> L) & 1ull);
        e &= seg;
        const uint64_t Q = (qt >> a) & seg & ~e;
        const uint64_t x = (prefix_xor(Q) ^ (str ? ~0ull : 0ull)) & seg;
        str = (uint32_t)((x >> (L - 1)) & 1ull);
        esc = esc_next;
        escd |= e << a;
        instr |= x << a;
        if (b == 64) break;
        a = b;
    }
    *escd_out = escd;
    *instr_out = instr;
    return esc | (str << 1);
}

__global__ void body_starts_kernel(BodyParams p) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= p.n_bodies) return;
    const uint64_t o = p.bodies[b].staged_off;
    atomicOr(p.starts + (o >> 6), 1ull << (o & 63));
}

__global__ void __launch_bounds__(256) json_trans_kernel(BodyParams p, uint64_t nblk) {
    __shared__ uint8_t lut[256];
    fill_class_lut(lut);
    __syncthreads();
    const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= nblk) return;
    const BlockBits bb = load_block(lut, p.text + 64 * k, false);
    const uint64_t S = p.starts[k];
    uint32_t t = 0;
    for (uint32_t s = 0; s < 4; ++s) {
        uint64_t e, x;
        t |= scan_block(bb.bs, bb.qt, S, s, &e, &x) << (2 * s);
    }
    p.trans[k] = (uint8_t)t;
}

__global__ void __launch_bounds__(256) json_classify_kernel(BodyParams p, uint64_t nblk) {
    __shared__ uint8_t lut[256];
    fill_class_lut(lut);
    __syncthreads();
    const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= nblk) return;
    const uint8_t* t = p.text + 64 * k;
    const BlockBits bb = load_block(lut, t, true);
    uint64_t escd, instr;
    scan_block(bb.bs, bb.qt, p.starts[k], p.carry[k] & 3u, &escd, &instr);
    const uint64_t Q = bb.qt & ~escd;
    const uint64_t sc = ~instr & ~bb.st & ~bb.ws & ~Q;  // bytes of scalars (and junk) outside strings
    uint64_t bad = (bb.ctl & instr) | (escd & ~bb.esc);
    for (uint64_t u = escd & bb.u & instr; u; u &= u - 1) {  // \uXXXX: four hex digits (the buffer has slack past the text)
        const int i = __ffsll((long long)u) - 1;
        bool ok = true;
        for (int j = 1; j <= 4; ++j) ok &= (lut[t[i + j]] & C_HEX) != 0;
        if (!ok) bad |= 1ull << i;
    }
    BlockMasks m;
    m.tok = (bb.st & ~instr) | (Q & instr) | sc;
    m.quote = Q;
    m.bs = bb.bs;
    m.bad = bad;
    p.masks[k] = m;
}

// a warp's window of 32 blocks of masks, lane l holding block wb + l
struct Window {
    uint64_t wb = ~0ull;
    BlockMasks m{};
};

__device__ __forceinline__ void window_at(const BodyParams& p, uint64_t nblk, Window& w, uint64_t blk, uint32_t lane) {
    if (w.wb != ~0ull && blk >= w.wb && blk < w.wb + 32) return;
    w.wb = blk;
    const uint64_t k = blk + lane;
    if (k < nblk) w.m = p.masks[k];
    else w.m = BlockMasks{0, 0, 0, 0};
}

// first token at or after p and before e (e when none)
__device__ uint64_t next_token(const BodyParams& p, uint64_t nblk, Window& w, uint64_t pos, uint64_t e, uint32_t lane) {
    while (pos < e) {
        window_at(p, nblk, w, pos >> 6, lane);
        const uint64_t rel = (pos >> 6) - w.wb;
        uint64_t m = lane < rel ? 0ull : w.m.tok;
        if (lane == rel) m &= ~0ull << (pos & 63);
        const uint32_t bal = __ballot_sync(~0u, m != 0);
        if (bal) {
            const int L = __ffs(bal) - 1;
            const uint64_t mm = __shfl_sync(~0u, m, L);
            const uint64_t at = (w.wb + L) * 64 + (uint64_t)(__ffsll((long long)mm) - 1);
            return at < e ? at : e;
        }
        pos = (w.wb + 32) * 64;
    }
    return e;
}

// the closing quote of a string whose characters start at pos (e when there is none before e); *bs: a backslash among
// the characters, *bad: a control character or a bad escape among them
__device__ uint64_t close_quote(const BodyParams& p, uint64_t nblk, Window& w, uint64_t pos, uint64_t e, uint32_t lane, bool* bs, bool* bad) {
    bool any_bs = false, any_bad = false;
    while (pos < e) {
        window_at(p, nblk, w, pos >> 6, lane);
        const uint64_t rel = (pos >> 6) - w.wb;
        uint64_t range = lane < rel ? 0ull : ~0ull;
        if (lane == rel) range = ~0ull << (pos & 63);
        const uint64_t m = w.m.quote & range;
        const uint32_t bal = __ballot_sync(~0u, m != 0);
        const uint32_t L = bal ? (uint32_t)(__ffs(bal) - 1) : 32u;
        uint64_t at = ~0ull;
        if (bal) {
            const uint64_t mm = __shfl_sync(~0u, m, L);
            at = (w.wb + L) * 64 + (uint64_t)(__ffsll((long long)mm) - 1);
        }
        if (lane > L) range = 0;
        if (lane == L) range &= (1ull << (at & 63)) - 1;
        any_bs |= __any_sync(~0u, (w.m.bs & range) != 0);
        any_bad |= __any_sync(~0u, (w.m.bad & range) != 0);
        if (bal) {
            *bs = any_bs;
            *bad = any_bad;
            return at < e ? at : e;
        }
        pos = (w.wb + 32) * 64;
    }
    *bs = any_bs;
    *bad = any_bad;
    return e;
}

// a scalar at t (Go's scanner: true, false, null, or -?(0|[1-9][0-9]*)(\.[0-9]+)?([eE][+-]?[0-9]+)?) ending at the first
// whitespace, structural character or quote.  Returns 0 invalid, 1 null, 2 another valid scalar; *end after it.
__device__ int scalar(const uint8_t* s, uint64_t t, uint64_t e, uint64_t* end) {
    uint64_t q = t;
    while (q < e) {
        const uint8_t c = s[q];
        if (c == ' ' || c == '\t' || c == '\n' || c == '\r' || c == '"' || c == '{' || c == '}' || c == '[' || c == ']' || c == ':' ||
            c == ',')
            break;
        ++q;
    }
    *end = q;
    const uint64_t n = q - t;
    const uint8_t* c = s + t;
    if (n == 4 && c[0] == 'n' && c[1] == 'u' && c[2] == 'l' && c[3] == 'l') return 1;
    if (n == 4 && c[0] == 't' && c[1] == 'r' && c[2] == 'u' && c[3] == 'e') return 2;
    if (n == 5 && c[0] == 'f' && c[1] == 'a' && c[2] == 'l' && c[3] == 's' && c[4] == 'e') return 2;
    uint64_t i = 0;
    auto digit = [&](uint64_t k) { return k < n && c[k] >= '0' && c[k] <= '9'; };
    if (i < n && c[i] == '-') ++i;
    if (!digit(i)) return 0;
    if (c[i] == '0') ++i;
    else
        while (digit(i)) ++i;
    if (i < n && c[i] == '.') {
        ++i;
        if (!digit(i)) return 0;
        while (digit(i)) ++i;
    }
    if (i < n && (c[i] == 'e' || c[i] == 'E')) {
        ++i;
        if (i < n && (c[i] == '+' || c[i] == '-')) ++i;
        if (!digit(i)) return 0;
        while (digit(i)) ++i;
    }
    return i == n ? 2 : 0;
}

__device__ __forceinline__ uint32_t hex4(const uint8_t* h) {
    uint32_t v = 0;
    for (int j = 0; j < 4; ++j) {
        const uint8_t c = h[j];
        v = v * 16 + (c <= '9' ? c - '0' : (c | 0x20) - 'a' + 10);
    }
    return v;
}

// A key's characters [a, b) unescaped into buf (UTF-8; a character of 3 bytes or more becomes one byte 0xFF, which no
// name holds).  Returns the length, or 13 when it is longer than any name.
__device__ uint32_t key_bytes(const uint8_t* s, uint64_t a, uint64_t b, uint8_t* buf) {
    uint32_t n = 0;
    for (uint64_t i = a; i < b;) {
        if (n > 12) return 13;
        uint8_t c = s[i];
        if (c != '\\') {
            buf[n++] = c;
            ++i;
            continue;
        }
        const uint8_t d = s[i + 1];
        i += 2;
        if (d == 'u') {
            const uint32_t v = hex4(s + i);
            i += 4;
            if (v < 0x80) buf[n++] = (uint8_t)v;
            else if (v < 0x800) {
                buf[n++] = (uint8_t)(0xC0 | (v >> 6));
                if (n <= 12) buf[n++] = (uint8_t)(0x80 | (v & 63));
            } else buf[n++] = 0xFF;
            continue;
        }
        buf[n++] = d == 'b' ? 8 : d == 'f' ? 12 : d == 'n' ? 10 : d == 'r' ? 13 : d == 't' ? 9 : d;
    }
    return n > 12 ? 13 : n;
}

// encoding/json's equalFoldRight for "entries" ('s' also matches U+017F, UTF-8 C5 BF)
__device__ bool is_entries(const uint8_t* k, uint32_t n) {
    const char* nm = "entries";
    uint32_t j = 0;
    for (int i = 0; i < 7; ++i) {
        if (j >= n) return false;
        const uint8_t sb = (uint8_t)nm[i], tb = k[j];
        if (tb < 0x80) {
            if ((tb & 0xDF) != (sb & 0xDF)) return false;
            ++j;
        } else {
            if (sb != 's' || j + 1 >= n || tb != 0xC5 || k[j + 1] != 0xBF) return false;
            j += 2;
        }
    }
    return j == n;
}

// asciiEqualFold: letters case-insensitively, every other byte exactly
__device__ bool is_name(const uint8_t* k, uint32_t n, const char* nm) {
    if (n != 10) return false;
    for (int i = 0; i < 10; ++i) {
        const uint8_t sb = (uint8_t)nm[i], tb = k[i];
        if (sb == tb) continue;
        if (!((sb >= 'a' && sb <= 'z')) || (sb & 0xDF) != (tb & 0xDF)) return false;
    }
    return true;
}

enum : uint32_t { EX_VALUE, EX_VALUE_OR_CLOSE, EX_KEY, EX_KEY_OR_CLOSE, EX_COLON, EX_COMMA_OR_CLOSE, EX_END };
enum : uint32_t { R_SKIP, R_TOP, R_ENTRIES, R_ELEM, R_LEAF, R_EXTRA };

// One warp per body: the grammar of the whole body and the spans of its entries.  Every lane runs the same walk; lane 0
// writes.
__global__ void __launch_bounds__(128) json_walk_kernel(BodyParams p, uint64_t nblk) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (b >= p.n_bodies) return;
    const BodyDesc d = p.bodies[b];
    const uint8_t* s = p.text;
    const uint64_t e = d.staged_off + d.len;
    Window w;
    uint64_t pos = d.staged_off;
    uint32_t depth = 0;
    uint64_t stk = 0;  // container kinds of depths 1..63 (1: object); deeper ones in p.stack, bit staged_off + depth
    bool resp = false, in_entries = false, in_elem = false;
    bool bad_json = false, bad_type = false;
    uint32_t entries_seen = 0, count = 0;
    uint64_t sp_off[2] = {~0ull, ~0ull};
    uint32_t sp_len[2] = {0, 0};
    uint8_t sp_esc = 0;
    uint32_t expect = EX_VALUE, role = R_TOP;
    uint8_t key[16];

    auto top_is_obj = [&]() -> bool {
        if (depth < 64) return (stk >> depth) & 1ull;
        const uint64_t bit = d.staged_off + depth;
        const uint32_t v = __shfl_sync(~0u, lane == 0 ? *((volatile uint32_t*)p.stack + (bit >> 5)) : 0u, 0);
        return (v >> (bit & 31)) & 1u;
    };
    auto push = [&](bool obj) {
        ++depth;
        if (depth < 64) {
            stk = obj ? stk | (1ull << depth) : stk & ~(1ull << depth);
            return;
        }
        const uint64_t bit = d.staged_off + depth;
        if (lane == 0) {
            if (obj) atomicOr(p.stack + (bit >> 5), 1u << (bit & 31));
            else atomicAnd(p.stack + (bit >> 5), ~(1u << (bit & 31)));
        }
        __syncwarp();
    };
    auto emit = [&]() {  // the element that just ended (an object or null) is entry `count` of the first entries array
        if (entries_seen == 1) {
            if (count < d.max && lane == 0) {
                const uint64_t slot = d.slot0 + count;
                p.s_off[0][slot] = sp_off[0];
                p.s_len[0][slot] = sp_len[0];
                p.s_off[1][slot] = sp_off[1];
                p.s_len[1][slot] = sp_len[1];
                p.s_esc[slot] = sp_esc;
            }
            ++count;
        }
        sp_off[0] = sp_off[1] = ~0ull;
        sp_len[0] = sp_len[1] = 0;
        sp_esc = 0;
    };
    auto after_value = [&]() { expect = depth == 0 ? EX_END : EX_COMMA_OR_CLOSE; };

    while (!bad_json) {
        const uint64_t t = next_token(p, nblk, w, pos, e, lane);
        if (t >= e) {
            bad_json = expect != EX_END;
            break;
        }
        const uint8_t c = s[t];
        pos = t + 1;
        if (expect == EX_END) {
            bad_json = true;
        } else if (expect == EX_COLON) {
            bad_json = c != ':';
            expect = EX_VALUE;
        } else if (expect == EX_COMMA_OR_CLOSE || ((expect == EX_VALUE_OR_CLOSE || expect == EX_KEY_OR_CLOSE) && (c == ']' || c == '}'))) {
            const bool obj = top_is_obj();
            if (expect == EX_COMMA_OR_CLOSE && c == ',') {
                expect = obj ? EX_KEY : EX_VALUE;
                role = (!obj && depth == 2 && in_entries) ? R_ELEM : R_SKIP;
            } else if (c == (obj ? '}' : ']') && (expect != EX_VALUE_OR_CLOSE || !obj) && (expect != EX_KEY_OR_CLOSE || obj)) {
                if (depth == 3 && in_elem) {
                    emit();
                    in_elem = false;
                }
                if (depth == 2) in_entries = false;
                --depth;
                after_value();
            } else {
                bad_json = true;
            }
        } else if (expect == EX_KEY || expect == EX_KEY_OR_CLOSE) {
            if (c != '"') {
                bad_json = true;
                break;
            }
            bool bs, bad;
            const uint64_t q = close_quote(p, nblk, w, t + 1, e, lane, &bs, &bad);
            if (q >= e || bad) {
                bad_json = true;
                break;
            }
            pos = q + 1;
            role = R_SKIP;
            if ((depth == 1 && resp) || (depth == 3 && in_elem)) {
                const uint32_t n = key_bytes(s, t + 1, q, key);
                if (depth == 1 && is_entries(key, n)) {
                    role = R_ENTRIES;
                    ++entries_seen;
                } else if (depth == 3 && is_name(key, n, "leaf_input")) {
                    role = R_LEAF;
                } else if (depth == 3 && is_name(key, n, "extra_data")) {
                    role = R_EXTRA;
                }
            }
            expect = EX_COLON;
        } else {  // a value
            if (c == '{' || c == '[') {
                const bool obj = c == '{';
                if (role == R_TOP && obj) resp = true;
                else if (role == R_ENTRIES && !obj) in_entries = true;  // a repeated array too: its types are checked
                else if (role == R_ELEM && obj) in_elem = true;
                else if (role != R_SKIP) bad_type = true;
                push(obj);
                expect = obj ? EX_KEY_OR_CLOSE : EX_VALUE_OR_CLOSE;
                role = (!obj && depth == 2 && in_entries) ? R_ELEM : R_SKIP;
            } else if (c == '"') {
                bool bs, bad;
                const uint64_t q = close_quote(p, nblk, w, t + 1, e, lane, &bs, &bad);
                if (q >= e || bad) {
                    bad_json = true;
                    break;
                }
                pos = q + 1;
                if (role == R_LEAF || role == R_EXTRA) {
                    const int k = role == R_EXTRA;
                    sp_off[k] = t + 1;
                    sp_len[k] = (uint32_t)(q - t - 1);
                    sp_esc = bs ? (uint8_t)(sp_esc | (1u << k)) : (uint8_t)(sp_esc & ~(1u << k));
                } else if (role != R_SKIP) {
                    bad_type = true;
                }
                after_value();
            } else if (c == ']' || c == '}' || c == ':' || c == ',') {
                bad_json = true;
            } else {
                uint64_t end;
                const int v = scalar(s, t, e, &end);
                if (v == 0) {
                    bad_json = true;
                    break;
                }
                pos = end;
                if (v == 1) {  // null: no entries, an empty element, an empty string
                    if (role == R_ELEM) emit();
                    if (role == R_LEAF || role == R_EXTRA) {
                        const int k = role == R_EXTRA;
                        sp_off[k] = ~0ull;
                        sp_len[k] = 0;
                        sp_esc &= (uint8_t)~(1u << k);
                    }
                } else if (role != R_SKIP) {
                    bad_type = true;
                }
                after_value();
            }
        }
    }
    if (lane == 0) {
        const uint8_t st = bad_json ? CTMR_BODY_BAD_JSON
                           : bad_type ? CTMR_BODY_BAD_TYPE
                           : entries_seen > 1 ? CTMR_BODY_REPEATED_ENTRIES
                           : count > d.max ? CTMR_BODY_TOO_MANY
                                           : CTMR_BODY_OK;
        p.body_status[b] = st;
        p.body_count[b] = st == CTMR_BODY_OK ? count : 0;
    }
}

// the entries of the OK bodies to dense positions: spans in the stage (offsets in the staged text), their offsets in the
// caller's text, the escape flags.  One warp per body.
__global__ void __launch_bounds__(128) json_compact_kernel(BodyParams p) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (b >= p.n_bodies) return;
    const BodyDesc d = p.bodies[b];
    const uint32_t cnt = p.body_count[b], base = p.body_base[b];
    for (uint32_t j = lane; j < cnt; j += 32) {
        const uint64_t slot = d.slot0 + j, o = base + j;
        for (int k = 0; k < 2; ++k) {
            const uint64_t off = p.s_off[k][slot];
            const bool none = off == ~0ull;
            p.off[k][o] = none ? 0 : off;
            p.len[k][o] = p.s_len[k][slot];
            p.abs_off[k][o] = none ? 0 : d.text_off + (off - d.staged_off);
            p.raw_len[k][o] = p.s_len[k][slot];
        }
        p.esc[o] = p.s_esc[slot];
    }
}

// one thread per string of the dense entries that held a backslash: unescaped into the spare half at the same offset
__global__ void __launch_bounds__(256) json_unescape_kernel(BodyParams p, uint64_t cap) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t n = p.body_base[p.n_bodies];
    if (i >= 2 * n || i >= 2 * cap) return;
    const uint64_t e = i >> 1;
    const int k = (int)(i & 1);
    if (!((p.esc[e] >> k) & 1u)) return;
    const uint8_t* s = p.text;
    const uint64_t a = p.off[k][e], z = a + p.len[k][e];
    uint8_t* dst = const_cast<uint8_t*>(p.text) + p.spare + a;
    uint32_t w = 0;
    for (uint64_t q = a; q < z;) {
        uint8_t c = s[q];
        uint32_t v;
        if (c != '\\') {
            v = c;
            ++q;
        } else {
            const uint8_t d = s[q + 1];
            q += 2;
            if (d == 'u') {
                v = hex4(s + q);
                q += 4;
            } else {
                v = d == 'b' ? 8 : d == 'f' ? 12 : d == 'n' ? 10 : d == 'r' ? 13 : d == 't' ? 9 : d;
            }
        }
        if (v == '\r' || v == '\n') continue;   // base64.StdEncoding skips them
        dst[w++] = v < 0x80 ? (uint8_t)v : (uint8_t)'!';  // outside the alphabet: the string stays BAD_BASE64
    }
    p.off[k][e] = p.spare + a;
    p.len[k][e] = w;
}

struct ComposeOp {  // the carry function of block x, then of block y
    __device__ __forceinline__ uint8_t operator()(uint8_t x, uint8_t y) const {
        uint32_t r = 0;
        for (uint32_t s = 0; s < 4; ++s) r |= ((y >> (2 * ((x >> (2 * s)) & 3u))) & 3u) << (2 * s);
        return (uint8_t)r;
    }
};
constexpr uint8_t kIdentity = 0xE4;  // state s -> s

}  // namespace

size_t json_scan_temp_bytes(uint64_t blocks, uint64_t bodies) {
    size_t a = 0, b = 0;
    cub::DeviceScan::ExclusiveScan(nullptr, a, (const uint8_t*)nullptr, (uint8_t*)nullptr, ComposeOp{}, kIdentity, (int)blocks);
    cub::DeviceScan::ExclusiveSum(nullptr, b, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)(bodies + 1));
    return a > b ? a : b;
}

cudaError_t launch_json_bodies(const BodyParams& p, uint64_t bytes, uint64_t sparse, void* temp, size_t temp_bytes, cudaStream_t s,
                               uint32_t* launches) {
    const uint64_t nblk = (bytes + 63) / 64;
    *launches = 0;
    if (!p.n_bodies) return cudaSuccess;
    cudaError_t err = cudaMemsetAsync(p.starts, 0, (nblk + 1) * 8, s);  // + 1: an empty body may start at the end
    if (err != cudaSuccess) return err;
    body_starts_kernel<<<(p.n_bodies + 255) / 256, 256, 0, s>>>(p);
    const uint32_t g = (uint32_t)((nblk + 255) / 256);
    if (nblk) {
        json_trans_kernel<<<g, 256, 0, s>>>(p, nblk);
        size_t tb = temp_bytes;
        err = cub::DeviceScan::ExclusiveScan(temp, tb, p.trans, p.carry, ComposeOp{}, kIdentity, (int)nblk, s);
        if (err != cudaSuccess) return err;
        json_classify_kernel<<<g, 256, 0, s>>>(p, nblk);
    }
    const uint32_t wg = (p.n_bodies + 3) / 4;
    json_walk_kernel<<<wg, 128, 0, s>>>(p, nblk);
    err = cudaMemsetAsync(p.body_count + p.n_bodies, 0, 4, s);
    if (err != cudaSuccess) return err;
    size_t tb = temp_bytes;
    err = cub::DeviceScan::ExclusiveSum(temp, tb, p.body_count, p.body_base, (int)(p.n_bodies + 1), s);
    if (err != cudaSuccess) return err;
    json_compact_kernel<<<wg, 128, 0, s>>>(p);
    if (sparse) json_unescape_kernel<<<(uint32_t)((2 * sparse + 255) / 256), 256, 0, s>>>(p, sparse);
    *launches = 9;  // starts, trans, scan, classify, walk, scan (two kernels each for cub counted once), compact, unescape
    return cudaGetLastError();
}

}  // namespace ctmr
