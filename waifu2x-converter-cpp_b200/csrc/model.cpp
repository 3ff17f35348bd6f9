// model.cpp -- model container + JSON model-file loader (host only, no CUDA).
//
// Stands in for w2xc::modelUtility::generateModelFromJSON (reference src/modelHandler.cpp:170-197),
// the Model constructor (src/modelHandler.hpp:48-71) and Model::loadModelFromJSONObject
// (src/modelHandler.cpp:74-115).  The reference parses with picojson, whose numbers go through
// strtod (include/picojson.h:788); std::from_chars<double> is the same correctly-rounded
// decimal->binary64 conversion without the locale dependence.  Weights are then narrowed
// double->float exactly as `writeMatrix.at<float>(r,c) = weightMatRow[c].get<double>()` does,
// biases stay double (src/modelHandler.hpp:30).
#include <atomic>
#include <charconv>
#include <cmath>
#include <cstring>
#include <fstream>
#include <memory>
#include <sstream>

#include "w2x_internal.h"

namespace w2x {

// ---- thread-local error string --------------------------------------------------------------
static thread_local std::string g_err;
int fail(int code, const char *fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_err = buf;
    return code;
}
const char *last_error_cstr() { return g_err.c_str(); }

// ---- fp16 helpers (host) --------------------------------------------------------------------
uint16_t f32_to_f16_rn(float f) {
    uint32_t x;
    std::memcpy(&x, &f, 4);
    uint32_t sign = (x >> 16) & 0x8000u;
    x &= 0x7fffffffu;
    if (x >= 0x7f800000u) return (uint16_t)(sign | 0x7c00u | (x > 0x7f800000u ? 0x200u : 0));
    if (x >= 0x477ff000u) {  // >= 65520 rounds to inf
        return (uint16_t)(sign | 0x7c00u);
    }
    if (x < 0x38800000u) {  // subnormal half (|f| < 2^-14) or zero
        if (x < 0x33000000u) return (uint16_t)sign;  // < 2^-25 -> 0 (2^-25 itself ties to even = 0)
        int e = (int)(x >> 23);                       // biased float exponent
        uint32_t m = (x & 0x7fffffu) | 0x800000u;     // 24-bit significand
        // value = m * 2^(e-150); half subnormal unit = 2^-24 -> q = m * 2^(e-126) = m >> (126-e)
        int shift = 126 - e;
        uint32_t q = m >> shift;
        uint32_t rem = m & ((1u << shift) - 1u);
        uint32_t half = 1u << (shift - 1);
        if (rem > half || (rem == half && (q & 1u))) q++;
        return (uint16_t)(sign | q);
    }
    uint32_t e = (x >> 23) - 112;  // half exponent
    uint32_t m = x & 0x7fffffu;
    uint32_t h = (e << 10) | (m >> 13);
    uint32_t rem = m & 0x1fffu;
    if (rem > 0x1000u || (rem == 0x1000u && (h & 1u))) h++;  // may carry into exponent: correct
    return (uint16_t)(sign | h);
}

uint16_t f32_to_bf16_rn(float f) {
    uint32_t x;
    std::memcpy(&x, &f, 4);
    if ((x & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((x >> 16) | 0x40u);   // NaN stays NaN
    if ((x & 0x7fffffffu) == 0x7f800000u) return (uint16_t)(x >> 16);             // +-inf
    x += 0x7fffu + ((x >> 16) & 1u);                                               // ties to even; may carry into the exponent
    if ((x & 0x7fffffffu) >= 0x7f800000u) x = (x & 0x80000000u) | 0x7f7f0000u;     // satfinite: a finite value stays finite
    return (uint16_t)(x >> 16);
}

float bf16_to_f32(uint16_t h) {
    const uint32_t x = (uint32_t)h << 16;
    float f;
    std::memcpy(&f, &x, 4);
    return f;
}

float f16_to_f32(uint16_t h) {
    uint32_t sign = (uint32_t)(h & 0x8000u) << 16;
    uint32_t e = (h >> 10) & 0x1f, m = h & 0x3ffu;
    uint32_t x;
    if (e == 0) {
        if (m == 0) x = sign;
        else {
            float v = std::ldexp((float)m, -24);
            std::memcpy(&x, &v, 4);
            x |= sign;
        }
    } else if (e == 31) x = sign | 0x7f800000u | (m << 13);
    else x = sign | ((e + 112) << 23) | (m << 13);
    float f;
    std::memcpy(&f, &x, 4);
    return f;
}

uint8_t f32_to_e4m3_rn(float f) {
    uint32_t x;
    std::memcpy(&x, &f, 4);
    const uint8_t sign = (uint8_t)((x >> 24) & 0x80u);
    float a = std::fabs(f);
    if (!(a == a)) return (uint8_t)(sign | 0x7f);       // NaN
    if (a >= 448.0f) return (uint8_t)(sign | 0x7e);     // satfinite
    if (a < 0.015625f) {                                // below the smallest normal 2^-6: subnormals, unit 2^-9
        int q = (int)std::nearbyint((double)a * 512.0); // FE_TONEAREST: ties to even; q == 8 encodes the first normal
        return (uint8_t)(sign | (uint8_t)q);
    }
    int e;
    float m = std::frexp(a, &e);                        // a = m * 2^e, m in [0.5, 1)
    e -= 1;                                             // a = (2m) * 2^e, 2m in [1, 2)
    int q = (int)std::nearbyint(((double)m * 2.0 - 1.0) * 8.0);
    if (q == 8) { q = 0; e += 1; }
    int enc = ((e + 7) << 3) | q;
    if (enc > 0x7e) enc = 0x7e;
    return (uint8_t)(sign | (uint8_t)enc);
}

// ---- a small JSON reader ----------------------------------------------------------------------
namespace {

struct JVal {
    enum T { Null, Bool, Num, Str, Arr, Obj } t = Null;
    double num = 0;
    bool b = false;
    bool flat = false;            // Arr whose elements are all numbers: kept in `nums` (a model file is 99.9 % such arrays: kernel rows, biases)
    std::string str;
    std::vector<JVal> arr;
    std::vector<double> nums;
    std::vector<std::pair<std::string, JVal>> obj;
    size_t size() const { return flat ? nums.size() : arr.size(); }
    bool is_num(size_t i) const { return flat || arr[i].t == Num; }
    double num_at(size_t i) const { return flat ? nums[i] : arr[i].num; }
    const JVal *get(const char *key) const {
        for (auto &kv : obj)
            if (kv.first == key) return &kv.second;
        return nullptr;
    }
};

struct Parser {
    const char *p, *end, *begin;
    std::string err;
    void ws() {
        while (p < end && (*p == ' ' || *p == '\t' || *p == '\n' || *p == '\r')) p++;
    }
    bool error(const char *what) {
        if (err.empty()) {
            std::ostringstream os;
            os << "syntax error at offset " << (p - begin) << ": " << what;
            err = os.str();
        }
        return false;
    }
    bool parse_string(std::string &out) {
        if (p >= end || *p != '"') return error("expected string");
        p++;
        while (p < end && *p != '"') {
            if (*p == '\\') {
                p++;
                if (p >= end) return error("bad escape");
                switch (*p) {
                    case '"': out += '"'; break;
                    case '\\': out += '\\'; break;
                    case '/': out += '/'; break;
                    case 'b': out += '\b'; break;
                    case 'f': out += '\f'; break;
                    case 'n': out += '\n'; break;
                    case 'r': out += '\r'; break;
                    case 't': out += '\t'; break;
                    case 'u': {
                        if (end - p < 5) return error("bad \\u escape");
                        unsigned cp = 0;
                        for (int i = 1; i <= 4; i++) {
                            char c = p[i];
                            cp <<= 4;
                            if (c >= '0' && c <= '9') cp |= (unsigned)(c - '0');
                            else if (c >= 'a' && c <= 'f') cp |= (unsigned)(c - 'a' + 10);
                            else if (c >= 'A' && c <= 'F') cp |= (unsigned)(c - 'A' + 10);
                            else return error("bad \\u escape");
                        }
                        p += 4;
                        if (cp < 0x80) out += (char)cp;
                        else if (cp < 0x800) { out += (char)(0xc0 | (cp >> 6)); out += (char)(0x80 | (cp & 0x3f)); }
                        else { out += (char)(0xe0 | (cp >> 12)); out += (char)(0x80 | ((cp >> 6) & 0x3f)); out += (char)(0x80 | (cp & 0x3f)); }
                        break;
                    }
                    default: return error("bad escape");
                }
                p++;
            } else out += *p++;
        }
        if (p >= end) return error("unterminated string");
        p++;
        return true;
    }
    // number token at p: the same scan + std::from_chars for every number of the file
    bool parse_number(double &d) {
        const char *q = p;
        if (*q == '-') q++;
        while (q < end && ((*q >= '0' && *q <= '9') || *q == '.' || *q == 'e' || *q == 'E' || *q == '+' || *q == '-')) q++;
        auto r = std::from_chars(p, q, d);
        if (r.ec != std::errc() || r.ptr != q) return false;
        p = q;
        return true;
    }
    bool parse_value(JVal &v, int depth) {
        if (depth > 64) return error("nesting too deep");
        ws();
        if (p >= end) return error("unexpected end of input");
        char c = *p;
        if (c == '[') {
            v.t = JVal::Arr;
            p++;
            ws();
            if (p < end && *p == ']') { p++; return true; }
            if (p < end && (*p == '-' || (*p >= '0' && *p <= '9'))) {
                // fast path: an array of numbers only.  Anything else in it (or a malformed number) rewinds to the generic path
                // below, which then produces exactly the diagnostics it always did.
                const char *rewind = p;
                for (;;) {
                    double d = 0;
                    if (p >= end || !(*p == '-' || (*p >= '0' && *p <= '9')) || !parse_number(d)) break;
                    v.nums.push_back(d);
                    ws();
                    if (p < end && *p == ',') { p++; ws(); continue; }
                    if (p < end && *p == ']') { p++; v.flat = true; return true; }
                    break;
                }
                v.nums.clear();
                p = rewind;
            }
            for (;;) {
                v.arr.emplace_back();
                if (!parse_value(v.arr.back(), depth + 1)) return false;
                ws();
                if (p < end && *p == ',') { p++; continue; }
                if (p < end && *p == ']') { p++; return true; }
                return error("expected ',' or ']'");
            }
        }
        if (c == '{') {
            v.t = JVal::Obj;
            p++;
            ws();
            if (p < end && *p == '}') { p++; return true; }
            for (;;) {
                ws();
                std::string key;
                if (!parse_string(key)) return false;
                ws();
                if (p >= end || *p != ':') return error("expected ':'");
                p++;
                v.obj.emplace_back(std::move(key), JVal());
                if (!parse_value(v.obj.back().second, depth + 1)) return false;
                ws();
                if (p < end && *p == ',') { p++; continue; }
                if (p < end && *p == '}') { p++; return true; }
                return error("expected ',' or '}'");
            }
        }
        if (c == '"') {
            v.t = JVal::Str;
            return parse_string(v.str);
        }
        if (c == 't' && end - p >= 4 && !std::strncmp(p, "true", 4)) { v.t = JVal::Bool; v.b = true; p += 4; return true; }
        if (c == 'f' && end - p >= 5 && !std::strncmp(p, "false", 5)) { v.t = JVal::Bool; v.b = false; p += 5; return true; }
        if (c == 'n' && end - p >= 4 && !std::strncmp(p, "null", 4)) { v.t = JVal::Null; p += 4; return true; }
        if (c == '-' || (c >= '0' && c <= '9')) {
            double d = 0;
            if (!parse_number(d)) return error("bad number");
            v.t = JVal::Num;
            v.num = d;
            return true;
        }
        return error("unexpected character");
    }
};

bool num_field(const JVal &o, const char *key, int &out) {
    const JVal *v = o.get(key);
    if (!v || v->t != JVal::Num) return false;
    if (!(v->num > -1e9 && v->num < 1e9)) return false;   // NaN / huge values: the cast below would be undefined behaviour
    out = static_cast<int>(v->num);  // static_cast<int>(get<double>()), src/modelHandler.hpp:50-52
    return true;
}

}  // namespace

static std::atomic<uint64_t> g_uid{1};

int parse_model_json(const char *path, w2x_model **out) {
    std::ifstream f(path, std::ios::binary);
    if (!f.is_open()) return fail(W2X_ERR_IO, "Error : couldn't open %s", path);
    std::string text((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
    Parser ps{text.data(), text.data() + text.size(), text.data(), {}};
    JVal root;
    if (!ps.parse_value(root, 0)) return fail(W2X_ERR_PARSE, "Error : PicoJSON Error : %s", ps.err.c_str());
    if (root.t != JVal::Arr)
        return fail(W2X_ERR_MODEL, "Error : model file %s : root is not an array of layer objects", path);
    auto m = std::make_unique<w2x_model>();
    if (root.flat) return fail(W2X_ERR_MODEL, "Error : model layer %zu is not an object", (size_t)0);
    for (size_t li = 0; li < root.arr.size(); li++) {
        const JVal &o = root.arr[li];
        if (o.t != JVal::Obj) return fail(W2X_ERR_MODEL, "Error : model layer %zu is not an object", li);
        Layer L;
        int kw = 0, kh = 0;
        if (!num_field(o, "nInputPlane", L.n_in) || !num_field(o, "nOutputPlane", L.n_out) ||
            !num_field(o, "kW", kw) || !num_field(o, "kH", kh))
            return fail(W2X_ERR_MODEL, "Error : model layer %zu : nInputPlane/nOutputPlane/kW/kH missing or not numbers", li);
        if (kw != kh)  // src/modelHandler.hpp:52-58 (the reference exits here)
            return fail(W2X_ERR_MODEL, "Error : Model-Constructor : \nkernel in model is not square.\nstop.");
        L.k = kw;
        if (L.n_in < 1 || L.n_out < 1 || L.k < 1)
            return fail(W2X_ERR_MODEL, "Error : model layer %zu : non-positive plane count or kernel size", li);
        const JVal *w = o.get("weight"), *b = o.get("bias");
        if (!w || w->t != JVal::Arr || !b || b->t != JVal::Arr)
            return fail(W2X_ERR_MODEL, "Error : model layer %zu : weight/bias missing or not arrays", li);
        // src/modelHandler.cpp:81-107: iterate weight[o][i], read kernelSize rows x kernelSize cols
        // (a `flat` array holds numbers where arrays are expected: the diagnostics are the ones the element-by-element walk gives)
        if ((int)w->size() != L.n_out)
            return fail(W2X_ERR_MODEL, "Error : model layer %zu : weight has %zu output planes, expected %d", li, w->size(), L.n_out);
        if (w->flat) return fail(W2X_ERR_MODEL, "Error : model layer %zu : weight[o] is not an array of %d input planes", li, L.n_in);
        L.w.resize((size_t)L.n_out * L.n_in * L.k * L.k);
        size_t idx = 0;
        for (const JVal &wo : w->arr) {
            if (wo.t != JVal::Arr || (int)wo.size() != L.n_in)
                return fail(W2X_ERR_MODEL, "Error : model layer %zu : weight[o] is not an array of %d input planes", li, L.n_in);
            if (wo.flat) return fail(W2X_ERR_MODEL, "Error : model layer %zu : kernel matrix has too few rows", li);
            for (const JVal &wi : wo.arr) {
                if (wi.t != JVal::Arr || (int)wi.size() < L.k)
                    return fail(W2X_ERR_MODEL, "Error : model layer %zu : kernel matrix has too few rows", li);
                if (wi.flat) return fail(W2X_ERR_MODEL, "Error : model layer %zu : kernel row has too few columns", li);
                for (int r = 0; r < L.k; r++) {
                    const JVal &row = wi.arr[(size_t)r];
                    if (row.t != JVal::Arr || (int)row.size() < L.k)
                        return fail(W2X_ERR_MODEL, "Error : model layer %zu : kernel row has too few columns", li);
                    for (int c = 0; c < L.k; c++) {
                        if (!row.is_num((size_t)c)) return fail(W2X_ERR_MODEL, "Error : model layer %zu : non-numeric weight", li);
                        L.w[idx++] = static_cast<float>(row.num_at((size_t)c));   // double -> float, cpp:96-97
                    }
                }
            }
        }
        if ((int)b->size() < L.n_out)
            return fail(W2X_ERR_MODEL, "Error : model layer %zu : bias has %zu entries, expected %d", li, b->size(), L.n_out);
        L.b.resize((size_t)L.n_out);
        for (int i = 0; i < L.n_out; i++) {
            if (!b->is_num((size_t)i)) return fail(W2X_ERR_MODEL, "Error : model layer %zu : non-numeric bias", li);
            L.b[(size_t)i] = b->num_at((size_t)i);                 // kept double, cpp:109-112
        }
        m->layers.push_back(std::move(L));
    }
    int rc = finalize_model(m.get());
    if (rc != W2X_OK) return rc;
    *out = m.release();
    return W2X_OK;
}

// ---- tensor-core operand packing ------------------------------------------------------------------
// Shared-memory image of one B block: n_out rows (one per output plane) of 32 fp16 values, K-major.
// Byte address of element (n, k) before swizzling: n*64 + 2k; the 16-byte unit index is then XORed
// with address bits [7,9) -- CUTLASS Swizzle<2,4,3>, the SWIZZLE_64B pattern of TMA / UMMA descriptors.
static inline size_t swizzled_offset(size_t logical, int row_bytes) {
    size_t mask = (size_t)(row_bytes / 16 - 1);  // 3 or 7
    return logical ^ (((logical >> 7) & mask) << 4);
}

static void pack_tc_layer(const Layer &L, TcPack &P) {
    // Blocks of 32 input channels (two K=16 MMA steps), rows of 64 B, SWIZZLE_64B, in the kernel's consumption
    // order: [32-channel block c (= one staged box of records)][tap][hi | lo].
    const int kc_a = 32;                       // channels per staged activation box (one record block)
    P.kc = 32;
    P.n_chunk = L.n_in / kc_a;
    P.kblocks = kc_a / 32;
    P.row_bytes = P.kc * 2;
    float mx = 0.f;
    for (float v : L.w) mx = std::fmax(mx, std::fabs(v));
    int e = 0;
    if (mx > 0.f) {
        e = (int)std::floor(std::log2(1024.0 / (double)mx));
        if (e < 0) e = 0;
        if (e > 14) e = 14;
    }
    P.wscale = std::ldexp(1.0f, e);
    const size_t block_elems = (size_t)L.n_out * P.kc;  // one (chunk, tap, kblock, part) block
    P.bytes.assign((size_t)P.n_chunk * 9 * P.kblocks * 2 * block_elems, 0);
    for (int c = 0; c < P.n_chunk; c++)
        for (int t = 0; t < 9; t++)
            for (int kb = 0; kb < P.kblocks; kb++) {
                const size_t blk = (((size_t)c * 9 + t) * P.kblocks + kb) * 2;
                uint16_t *hi = P.bytes.data() + (blk + 0) * block_elems;
                uint16_t *lo = P.bytes.data() + (blk + 1) * block_elems;
                for (int n = 0; n < L.n_out; n++)
                    for (int k = 0; k < P.kc; k++) {
                        int ci = c * kc_a + kb * 32 + k;
                        float w = L.w[((size_t)n * L.n_in + ci) * 9 + t] * P.wscale;  // exact (power of two)
                        uint16_t h = f32_to_f16_rn(w);
                        uint16_t l = f32_to_f16_rn(w - f16_to_f32(h));              // exact difference
                        size_t off = swizzled_offset((size_t)n * P.row_bytes + 2 * (size_t)k, P.row_bytes) / 2;
                        hi[off] = h;
                        lo[off] = l;
                    }
            }
}

// The bf16x3 operand image of the same layer (see TcPack::bytes_bf16): the f16x3 layout and swizzle, bf16 halves at wscale 1.
// bf16 has fp32's exponent range, so no power-of-two lift is needed and every finite weight packs.
static void pack_tc_layer_bf16(const Layer &L, TcPack &P) {
    const int kc = 32, n_chunk = L.n_in / kc, row_bytes = kc * 2;
    const size_t block_elems = (size_t)L.n_out * kc;
    P.bytes_bf16.assign((size_t)n_chunk * 9 * 2 * block_elems, 0);
    for (int c = 0; c < n_chunk; c++)
        for (int t = 0; t < 9; t++) {
            uint16_t *hi = P.bytes_bf16.data() + ((size_t)c * 9 + t) * 2 * block_elems, *lo = hi + block_elems;
            for (int n = 0; n < L.n_out; n++)
                for (int k = 0; k < kc; k++) {
                    const float w = L.w[((size_t)n * L.n_in + c * kc + k) * 9 + t];
                    const uint16_t h = f32_to_bf16_rn(w);
                    const size_t off = swizzled_offset((size_t)n * row_bytes + 2 * (size_t)k, row_bytes) / 2;
                    hi[off] = h;
                    lo[off] = f32_to_bf16_rn(w - bf16_to_f32(h));                  // exact difference
                }
        }
}

// The "f8" operand image of the same layer (see TcPack::bytes8).
static inline size_t swizzle32(size_t logical) { return logical ^ (((logical >> 7) & 1) << 4); }

static void pack_tc_layer_f8(const Layer &L, TcPack &P) {
    const int kc_a = 32;                       // channels per staged activation box (one record block)
    const size_t blk16 = (size_t)L.n_out * 64, blk8 = (size_t)L.n_out * 32, stage = blk16 + 2 * blk8;
    P.bytes8.assign((size_t)P.n_chunk * 9 * P.kblocks * stage, 0);
    const float up = std::ldexp(1.0f, F8_C), down = std::ldexp(1.0f, -F8_A);
    for (int c = 0; c < P.n_chunk; c++)
        for (int t = 0; t < 9; t++)
            for (int kb = 0; kb < P.kblocks; kb++) {
                uint8_t *base = P.bytes8.data() + (((size_t)c * 9 + t) * P.kblocks + kb) * stage;
                uint16_t *wh16 = reinterpret_cast<uint16_t *>(base);
                uint8_t *wh8 = base + blk16, *wl8 = wh8 + blk8;
                for (int n = 0; n < L.n_out; n++)
                    for (int k = 0; k < 32; k++) {
                        int ci = c * kc_a + kb * 32 + k;
                        float w = L.w[((size_t)n * L.n_in + ci) * 9 + t] * P.wscale;
                        uint16_t h = f32_to_f16_rn(w);
                        float hf = f16_to_f32(h);
                        wh16[swizzled_offset((size_t)n * 64 + 2 * (size_t)k, 64) / 2] = h;
                        wh8[swizzle32((size_t)n * 32 + (size_t)k)] = f32_to_e4m3_rn(hf * down);
                        wl8[swizzle32((size_t)n * 32 + (size_t)k)] = f32_to_e4m3_rn((w - hf) * up);
                    }
            }
}

// Operand images of the row-strip design (narrow layers, Cin and Cout <= 64; no kernel of this build reads them, the
// 16x16-tile kernel runs every layer; tests/test_strip_kernel_model.py checks them against the weights): per
// (32-channel chunk c, tap column kx) ONE stage whose rows are ky-major, row = ky * n_out + n, so that an N = 3*n_out MMA
// multiplies one staged input row by the three taps W(ky = 0..2, kx) at once:
//   strip   (f16x3): [wh: 3*n_out rows x 64 B, SWIZZLE_64B][wl: same]
//   strip8  (f8)   : [wh: 3*n_out rows x 64 B, SWIZZLE_64B][wh8 : 3*n_out rows x 32 B, SWIZZLE_32B][wl8: same]
// Same values (wscale, fp16 / e4m3 roundings) as the tap-major packs above.
static void pack_tc_layer_strip(const Layer &L, TcPack &P) {
    if (L.n_in > 64 || L.n_out > 64) return;
    const int nch = L.n_in / 32, nrows = 3 * L.n_out;
    const size_t stage = (size_t)nrows * 128;
    P.strip.assign((size_t)nch * 3 * stage, 0);
    P.strip8.assign((size_t)nch * 3 * stage, 0);
    const float up = std::ldexp(1.0f, F8_C), down = std::ldexp(1.0f, -F8_A);
    for (int c = 0; c < nch; c++)
        for (int kx = 0; kx < 3; kx++) {
            uint8_t *s16 = P.strip.data() + ((size_t)c * 3 + kx) * stage, *s8 = P.strip8.data() + ((size_t)c * 3 + kx) * stage;
            uint16_t *wh = reinterpret_cast<uint16_t *>(s16), *wl = reinterpret_cast<uint16_t *>(s16 + (size_t)nrows * 64);
            uint16_t *wh_f8 = reinterpret_cast<uint16_t *>(s8);
            uint8_t *wh8 = s8 + (size_t)nrows * 64, *wl8 = wh8 + (size_t)nrows * 32;
            for (int ky = 0; ky < 3; ky++)
                for (int n = 0; n < L.n_out; n++)
                    for (int k = 0; k < 32; k++) {
                        const size_t row = (size_t)ky * L.n_out + n;
                        const float w = L.w[((size_t)n * L.n_in + (c * 32 + k)) * 9 + ky * 3 + kx] * P.wscale;   // exact (power of two)
                        const uint16_t h = f32_to_f16_rn(w);
                        const float hf = f16_to_f32(h);
                        const size_t o16 = swizzled_offset(row * 64 + 2 * (size_t)k, 64) / 2, o8 = swizzle32(row * 32 + (size_t)k);
                        wh[o16] = h;
                        wl[o16] = f32_to_f16_rn(w - hf);
                        wh_f8[o16] = h;
                        wh8[o8] = f32_to_e4m3_rn(hf * down);
                        wl8[o8] = f32_to_e4m3_rn((w - hf) * up);
                    }
        }
}

// Whether the tensor-core operand images can hold the layer's weights: wscale is never below 1, so a weight of
// |w| >= 65520 (or a non-finite one) would pack as an fp16 infinity.
static bool tc_packable(const Layer &L) {
    for (float v : L.w)
        if (!(std::fabs(v) < 65520.f)) return false;
    return true;
}
// ... and the bf16x3 image: every finite weight.
static bool tc_packable_bf16(const Layer &L) {
    for (float v : L.w)
        if (!std::isfinite(v)) return false;
    return true;
}

int finalize_model(w2x_model *m) {
    if (m->layers.empty()) return fail(W2X_ERR_MODEL, "Error : model has no layers");
    for (size_t i = 0; i < m->layers.size(); i++) {
        const Layer &L = m->layers[i];
        if (L.k != 3)
            return fail(W2X_ERR_MODEL, "Error : model layer %zu : kernel size %d is not supported (only 3x3)", i, L.k);
        if (i > 0 && L.n_in != m->layers[i - 1].n_out)
            return fail(W2X_ERR_MODEL, "Error : model layer %zu : nInputPlane %d does not match previous nOutputPlane %d",
                        i, L.n_in, m->layers[i - 1].n_out);
    }
    // tensor-core eligibility: 1 -> C1 -> ... -> Cn -> 1 with every inner width in {32, 64, 128} and every inner layer packable
    // (fp16 images: finite weights below 65520; bf16x3: finite weights)
    auto okc = [](int c) { return c == 32 || c == 64 || c == 128; };
    size_t n = m->layers.size();
    const bool shape = n >= 3 && m->layers.front().n_in == 1 && m->layers.back().n_out == 1 &&
                       okc(m->layers.front().n_out) && okc(m->layers.back().n_in);
    bool ok = shape, ok_bf16 = shape;
    for (size_t i = 1; i + 1 < n; i++) {
        const bool c = okc(m->layers[i].n_in) && okc(m->layers[i].n_out);
        ok = ok && c && tc_packable(m->layers[i]);
        ok_bf16 = ok_bf16 && c && tc_packable_bf16(m->layers[i]);
    }
    m->tc_eligible = ok;
    m->tc_eligible_bf16 = ok_bf16;
    m->tc.assign(n, TcPack());
    for (size_t i = 0; i < n; i++) {
        const Layer &L = m->layers[i];
        if (!okc(L.n_in) || !okc(L.n_out)) continue;
        if (tc_packable(L)) {
            pack_tc_layer(L, m->tc[i]);
            pack_tc_layer_f8(L, m->tc[i]);
        }
        if (tc_packable_bf16(L)) pack_tc_layer_bf16(L, m->tc[i]);
    }
    m->uid = g_uid.fetch_add(1);
    return W2X_OK;
}

}  // namespace w2x

// ---- C ABI: model container ---------------------------------------------------------------------
namespace w2x { const char *last_error_cstr(); }

extern "C" {

const char *w2x_last_error(void) { return w2x::last_error_cstr(); }
const char *w2x_version(void) { return "1.0.0-b200.1"; }

int w2x_model_load_json(const char *path, w2x_model **out_model) {
    if (!path || !out_model) return w2x::fail(W2X_ERR_ARG, "w2x_model_load_json: NULL argument");
    *out_model = nullptr;
    try {
        return w2x::parse_model_json(path, out_model);
    } catch (const std::bad_alloc &) {
        return w2x::fail(W2X_ERR_NOMEM, "w2x_model_load_json: out of memory");
    } catch (const std::exception &e) {          // nothing may cross the C ABI
        return w2x::fail(W2X_ERR_PARSE, "w2x_model_load_json: %s", e.what());
    } catch (...) {
        return w2x::fail(W2X_ERR_PARSE, "w2x_model_load_json: unexpected failure");
    }
}

int w2x_model_create(int n_layers, const int *n_in, const int *n_out, const float *const *weights,
                     const double *const *biases, w2x_model **out_model) {
    if (n_layers < 1 || !n_in || !n_out || !weights || !biases || !out_model)
        return w2x::fail(W2X_ERR_ARG, "w2x_model_create: bad argument");
    *out_model = nullptr;
    auto m = std::make_unique<w2x_model>();
    for (int i = 0; i < n_layers; i++) {
        if (n_in[i] < 1 || n_out[i] < 1 || !weights[i] || !biases[i])
            return w2x::fail(W2X_ERR_ARG, "w2x_model_create: bad layer %d", i);
        w2x::Layer L;
        L.n_in = n_in[i];
        L.n_out = n_out[i];
        L.k = 3;
        L.w.assign(weights[i], weights[i] + (size_t)L.n_in * L.n_out * 9);
        L.b.assign(biases[i], biases[i] + L.n_out);
        m->layers.push_back(std::move(L));
    }
    int rc = w2x::finalize_model(m.get());
    if (rc != W2X_OK) return rc;
    *out_model = m.release();
    return W2X_OK;
}

void w2x_model_free(w2x_model *model) { delete model; }

int w2x_model_layer_count(const w2x_model *model) { return model ? (int)model->layers.size() : -W2X_ERR_ARG; }

int w2x_model_layer_dims(const w2x_model *model, int layer, int *n_in, int *n_out, int *k) {
    if (!model || layer < 0 || layer >= (int)model->layers.size())
        return w2x::fail(W2X_ERR_ARG, "w2x_model_layer_dims: bad model or layer index");
    const w2x::Layer &L = model->layers[(size_t)layer];
    if (n_in) *n_in = L.n_in;
    if (n_out) *n_out = L.n_out;
    if (k) *k = L.k;
    return W2X_OK;
}

int w2x_model_layer_params(const w2x_model *model, int layer, const float **weights, const double **biases) {
    if (!model || layer < 0 || layer >= (int)model->layers.size())
        return w2x::fail(W2X_ERR_ARG, "w2x_model_layer_params: bad model or layer index");
    const w2x::Layer &L = model->layers[(size_t)layer];
    if (weights) *weights = L.w.data();
    if (biases) *biases = L.b.data();
    return W2X_OK;
}

// Probe hook (not part of the stable ABI): the tensor-core operand image of one layer, for the packing tests.
W2X_API int w2x_debug_tc_pack(const w2x_model *model, int layer, const uint16_t **data, size_t *n_elems, int *kc,
                              int *n_chunk, float *wscale, int *kblocks) {
    if (!model || layer < 0 || layer >= (int)model->tc.size())
        return w2x::fail(W2X_ERR_ARG, "w2x_debug_tc_pack: bad model or layer index");
    const w2x::TcPack &P = model->tc[(size_t)layer];
    if (data) *data = P.bytes.data();
    if (n_elems) *n_elems = P.bytes.size();
    if (kc) *kc = P.kc;
    if (n_chunk) *n_chunk = P.n_chunk;
    if (wscale) *wscale = P.wscale;
    if (kblocks) *kblocks = P.kblocks;
    return W2X_OK;
}

// f8 = 0: TcPack::strip ([wh | wl]), f8 = 1: TcPack::strip8 ([wh | wh8 | wl8]); empty for layers outside the row-strip design.
W2X_API int w2x_debug_tc_strip(const w2x_model *model, int layer, int f8, const uint8_t **data, size_t *n_bytes) {
    if (!model || layer < 0 || layer >= (int)model->tc.size())
        return w2x::fail(W2X_ERR_ARG, "w2x_debug_tc_strip: bad model or layer index");
    // packed on the first request: no kernel reads these images, so loading a model does not build them
    w2x::TcPack &P = const_cast<w2x::TcPack &>(model->tc[(size_t)layer]);
    if (P.strip.empty() && !P.bytes.empty()) pack_tc_layer_strip(model->layers[(size_t)layer], P);
    const std::vector<uint8_t> &v = f8 ? P.strip8 : P.strip;
    if (data) *data = v.data();
    if (n_bytes) *n_bytes = v.size();
    return W2X_OK;
}

// The bf16x3 operand image of one layer (TcPack::bytes_bf16: bf16 bit patterns in the f16x3 layout, wscale 1); empty for layers
// outside the tensor-core shapes or with a non-finite weight.
W2X_API int w2x_debug_tc_pack_bf16(const w2x_model *model, int layer, const uint16_t **data, size_t *n_elems) {
    if (!model || layer < 0 || layer >= (int)model->tc.size())
        return w2x::fail(W2X_ERR_ARG, "w2x_debug_tc_pack_bf16: bad model or layer index");
    if (data) *data = model->tc[(size_t)layer].bytes_bf16.data();
    if (n_elems) *n_elems = model->tc[(size_t)layer].bytes_bf16.size();
    return W2X_OK;
}

W2X_API int w2x_debug_tc_pack8(const w2x_model *model, int layer, const uint8_t **data, size_t *n_bytes) {
    if (!model || layer < 0 || layer >= (int)model->tc.size())
        return w2x::fail(W2X_ERR_ARG, "w2x_debug_tc_pack8: bad model or layer index");
    if (data) *data = model->tc[(size_t)layer].bytes8.data();
    if (n_bytes) *n_bytes = model->tc[(size_t)layer].bytes8.size();
    return W2X_OK;
}

}  // extern "C"
