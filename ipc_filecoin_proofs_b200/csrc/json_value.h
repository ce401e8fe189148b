// json_value.h — the JSON value parser of the host-side readers (csrc/bundle_parse.cpp, csrc/rpc_parse.cpp, csrc/rpc_blocks_parse.cpp): a DOM of the text in
// serde_json's grammar (RFC 8259, escapes decoded, number literals kept as text) and the field readers the readers share. Plain C++,
// built with g++; every reader includes it into its own anonymous namespace. A failed field read throws Fail with its status.
#pragma once
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <string>
#include <utility>
#include <vector>

#include "../../include/ipcfp.h"

namespace {

struct JV {
    enum T { NUL, BOOL, NUM, STR, ARR, OBJ } t = NUL;
    bool b = false;
    std::string s;   // NUM: the literal's text, STR: the decoded string
    std::vector<JV> a;
    std::vector<std::pair<std::string, JV>> o;
    const JV* get(const char* k) const {
        if (t != OBJ) return nullptr;
        for (auto& kv : o) if (kv.first == k) return &kv.second;
        return nullptr;
    }
};

struct Parser {
    const char* p;
    const char* e;
    bool ok = true;
    void ws() { while (p < e && (*p == ' ' || *p == '\t' || *p == '\n' || *p == '\r')) p++; }
    bool lit(const char* w) {
        size_t n = strlen(w);
        if ((size_t)(e - p) < n || memcmp(p, w, n)) return false;
        p += n;
        return true;
    }
    static void utf8(std::string& o, uint32_t c) {
        if (c < 0x80) o.push_back((char)c);
        else if (c < 0x800) { o.push_back((char)(0xc0 | (c >> 6))); o.push_back((char)(0x80 | (c & 63))); }
        else if (c < 0x10000) { o.push_back((char)(0xe0 | (c >> 12))); o.push_back((char)(0x80 | ((c >> 6) & 63))); o.push_back((char)(0x80 | (c & 63))); }
        else { o.push_back((char)(0xf0 | (c >> 18))); o.push_back((char)(0x80 | ((c >> 12) & 63))); o.push_back((char)(0x80 | ((c >> 6) & 63))); o.push_back((char)(0x80 | (c & 63))); }
    }
    bool hex4(uint32_t& v) {
        if (e - p < 4) return false;
        v = 0;
        for (int i = 0; i < 4; i++) {
            char c = *p++;
            uint32_t d = c >= '0' && c <= '9' ? c - '0' : c >= 'a' && c <= 'f' ? c - 'a' + 10 : c >= 'A' && c <= 'F' ? c - 'A' + 10 : 99;
            if (d == 99) return false;
            v = v * 16 + d;
        }
        return true;
    }
    bool str(std::string& out) {
        if (p >= e || *p != '"') return false;
        p++;
        const char* run = p;
        for (;;) {
            if (p >= e) return false;
            unsigned char c = (unsigned char)*p;
            if (c == '"') { out.append(run, p - run); p++; return true; }
            if (c < 0x20) return false;
            if (c != '\\') { p++; continue; }
            out.append(run, p - run);
            p++;
            if (p >= e) return false;
            char x = *p++;
            switch (x) {
                case '"': out.push_back('"'); break;
                case '\\': out.push_back('\\'); break;
                case '/': out.push_back('/'); break;
                case 'b': out.push_back('\b'); break;
                case 'f': out.push_back('\f'); break;
                case 'n': out.push_back('\n'); break;
                case 'r': out.push_back('\r'); break;
                case 't': out.push_back('\t'); break;
                case 'u': {
                    uint32_t v;
                    if (!hex4(v)) return false;
                    if (v >= 0xd800 && v < 0xdc00) {   // surrogate pair
                        uint32_t w;
                        if (e - p < 6 || p[0] != '\\' || p[1] != 'u') return false;
                        p += 2;
                        if (!hex4(w) || w < 0xdc00 || w > 0xdfff) return false;
                        v = 0x10000 + ((v - 0xd800) << 10) + (w - 0xdc00);
                    } else if (v >= 0xdc00 && v <= 0xdfff) return false;
                    utf8(out, v);
                    break;
                }
                default: return false;
            }
            run = p;
        }
    }
    bool value(JV& v, int depth) {
        if (depth > 64) return false;
        ws();
        if (p >= e) return false;
        char c = *p;
        if (c == '{') {
            p++;
            v.t = JV::OBJ;
            ws();
            if (p < e && *p == '}') { p++; return true; }
            for (;;) {
                ws();
                std::string k;
                if (!str(k)) return false;
                ws();
                if (p >= e || *p != ':') return false;
                p++;
                v.o.emplace_back(std::move(k), JV());
                if (!value(v.o.back().second, depth + 1)) return false;
                ws();
                if (p < e && *p == ',') { p++; continue; }
                if (p < e && *p == '}') { p++; return true; }
                return false;
            }
        }
        if (c == '[') {
            p++;
            v.t = JV::ARR;
            ws();
            if (p < e && *p == ']') { p++; return true; }
            for (;;) {
                v.a.emplace_back();
                if (!value(v.a.back(), depth + 1)) return false;
                ws();
                if (p < e && *p == ',') { p++; continue; }
                if (p < e && *p == ']') { p++; return true; }
                return false;
            }
        }
        if (c == '"') { v.t = JV::STR; return str(v.s); }
        if (c == 't') { v.t = JV::BOOL; v.b = true; return lit("true"); }
        if (c == 'f') { v.t = JV::BOOL; v.b = false; return lit("false"); }
        if (c == 'n') { v.t = JV::NUL; return lit("null"); }
        if (c == '-' || (c >= '0' && c <= '9')) {
            const char* s0 = p;
            if (*p == '-') p++;
            if (p >= e || *p < '0' || *p > '9') return false;
            if (*p == '0') p++; else while (p < e && *p >= '0' && *p <= '9') p++;
            if (p < e && *p == '.') { p++; if (p >= e || *p < '0' || *p > '9') return false; while (p < e && *p >= '0' && *p <= '9') p++; }
            if (p < e && (*p == 'e' || *p == 'E')) { p++; if (p < e && (*p == '+' || *p == '-')) p++; if (p >= e || *p < '0' || *p > '9') return false; while (p < e && *p >= '0' && *p <= '9') p++; }
            v.t = JV::NUM;
            v.s.assign(s0, p - s0);
            return true;
        }
        return false;
    }
};

struct Fail { ipcfp_status st; };
[[noreturn]] void bad(ipcfp_status st = IPCFP_ERR_INVALID_ARG) { throw Fail{st}; }

const JV& need(const JV& o, const char* k, JV::T t) {
    const JV* v = o.get(k);
    if (!v || v->t != t) bad();
    return *v;
}
uint64_t u64_of(const JV& v) {   // serde: u64 fields take non-negative integer literals only
    if (v.t != JV::NUM || v.s.empty() || v.s.size() > 20) bad();
    uint64_t x = 0;
    for (char c : v.s) {
        if (c < '0' || c > '9') bad();
        uint64_t d = (uint64_t)(c - '0');
        if (x > (UINT64_MAX - d) / 10) bad();
        x = x * 10 + d;
    }
    return x;
}
int64_t i64_of(const JV& v) {   // ChainEpoch = i64
    if (v.t != JV::NUM || v.s.empty()) bad();
    bool neg = v.s[0] == '-';
    JV m;
    m.t = JV::NUM;
    m.s = neg ? v.s.substr(1) : v.s;
    uint64_t a = u64_of(m);
    if (neg) { if (a > (uint64_t)INT64_MAX + 1) bad(); return (int64_t)(0 - a); }
    if (a > (uint64_t)INT64_MAX) bad();
    return (int64_t)a;
}
// "b" + base32 lower, no padding → bytes; the C ABI carries 38-byte CIDs only
void cid_of_string(const std::string& s, uint8_t out[IPCFP_CID_LEN]) {
    if (s.empty() || s[0] != 'b') bad(IPCFP_ERR_UNSUPPORTED);
    std::vector<uint8_t> raw;
    uint32_t acc = 0;
    int bits = 0;
    for (size_t i = 1; i < s.size(); i++) {
        char c = s[i];
        uint32_t d = c >= 'a' && c <= 'z' ? (uint32_t)(c - 'a') : c >= '2' && c <= '7' ? (uint32_t)(c - '2' + 26) : 99;
        if (d == 99) bad();
        acc = (acc << 5) | d;
        bits += 5;
        if (bits >= 8) { raw.push_back((uint8_t)(acc >> (bits - 8))); bits -= 8; acc &= (1u << bits) - 1; }
    }
    if (acc != 0) bad();   // non-zero padding bits
    if (raw.size() != IPCFP_CID_LEN) bad(IPCFP_ERR_UNSUPPORTED);
    memcpy(out, raw.data(), IPCFP_CID_LEN);
}
void unbase64(const std::string& s, std::vector<uint8_t>& out) {   // standard alphabet, padding required (base64::STANDARD)
    if (s.size() % 4) bad();
    auto d = [](char c) -> uint32_t {
        return c >= 'A' && c <= 'Z' ? (uint32_t)(c - 'A') : c >= 'a' && c <= 'z' ? (uint32_t)(c - 'a' + 26) : c >= '0' && c <= '9' ? (uint32_t)(c - '0' + 52)
               : c == '+' ? 62u : c == '/' ? 63u : 99u;
    };
    for (size_t i = 0; i < s.size(); i += 4) {
        const bool last = i + 4 == s.size();
        uint32_t a = d(s[i]), b = d(s[i + 1]);
        if (a == 99 || b == 99) bad();
        const bool p3 = s[i + 3] == '=', p2 = s[i + 2] == '=';
        if ((p2 || p3) && !last) bad();
        if (p2 && !p3) bad();
        uint32_t c = p2 ? 0 : d(s[i + 2]), e = p3 ? 0 : d(s[i + 3]);
        if (c == 99 || e == 99) bad();
        uint32_t v = (a << 18) | (b << 12) | (c << 6) | e;
        out.push_back((uint8_t)(v >> 16));
        if (!p2) out.push_back((uint8_t)(v >> 8)); else if (b & 15) bad();          // canonical: unused bits are zero
        if (!p3) out.push_back((uint8_t)v); else if (!p2 && (c & 3)) bad();
    }
}

}  // namespace
