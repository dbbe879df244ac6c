// jpeg_decode_host.cpp — the host half of the baseline JPEG decoder: marker parsing, table building and the
// entropy range, as pixo::decode::decode_jpeg does them (src/decode/jpeg.rs).  Headers are a few hundred bytes,
// so they are parsed here; the scan, the IDCT and the colour conversion run on the device (jpeg_decode.cu).
#include "jpeg_decode_host.hpp"

#include <string.h>

#include <algorithm>

namespace pixo {

uint64_t JdecParsed::blocks() const
{
    uint64_t b = 0;
    for (uint32_t c = 0; c < ncomp; ++c) b += plane_w(c) / 8 * (plane_h(c) / 8);
    return b;
}

// HuffmanTable::build (src/decode/jpeg.rs:77-147).  Code lengths come from the counts; codes are kept as u16, as
// pixo keeps them, so an oversubscribed table builds the same lookup and max_code as it does there.
static void build_huff(const uint8_t bits[16], const uint8_t *values, uint32_t nvalues, JdecHuff &t,
                       std::vector<uint8_t> &vals)
{
    memset(&t, 0, sizeof t);
    vals.assign(values, values + nvalues);
    t.nvalues = nvalues;
    std::vector<uint8_t> size;
    std::vector<uint16_t> code;
    for (int i = 0; i < 16; ++i) size.insert(size.end(), bits[i], (uint8_t)(i + 1));
    uint32_t c = 0;
    uint8_t si = size.empty() ? 0 : size[0];
    for (uint8_t s : size) {
        for (; s > si; ++si) c <<= 1;
        code.push_back((uint16_t)c);
        ++c;
    }
    uint32_t idx = 0;
    t.max_code[0] = -1;
    for (int i = 1; i <= 16; ++i) {
        if (bits[i - 1]) {
            t.val_offset[i] = (int32_t)(idx - code[idx]);
            idx += bits[i - 1];
            t.max_code[i] = code[idx - 1];
        } else {
            t.max_code[i] = -1;
        }
    }
    uint32_t k = 0;
    for (int len = 1; len <= 16; ++len)
        for (int j = 0; j < bits[len - 1]; ++j, ++k) {
            if (len > 8) continue;
            const uint32_t fill = 8 - len, base = (uint32_t)code[k] << fill;
            for (uint32_t i = 0; i < (1u << fill); ++i)
                if ((base | i) < 256) t.lookup[base | i] = (uint16_t)(values[k] | (len << 8));
        }
}

static void empty_huff(JdecHuff &t)
{
    memset(&t, 0, sizeof t);
    for (int i = 0; i < 17; ++i) t.max_code[i] = -1;
}

size_t jdec_entropy_end(const uint8_t *d, size_t n)
{
    if (n < 2) return n;
    size_t i = 0;
    while (i < n - 1) {
        if (d[i] == 0xFF && d[i + 1] != 0x00 && d[i + 1] != 0xFF) {
            if (d[i + 1] >= 0xD0 && d[i + 1] <= 0xD7) {
                i += 2;
                continue;
            }
            return i;
        }
        ++i;
    }
    return n;
}

namespace {

struct Parser {
    const uint8_t *d;
    size_t n, pos = 2;
    JdecParsed &p;

    // read_marker (:253-292)
    bool marker(uint8_t &m, const uint8_t *&seg, size_t &len)
    {
        while (pos < n && d[pos] != 0xFF) ++pos;
        while (pos < n && d[pos] == 0xFF) ++pos;
        if (pos >= n) return decode_fail(p.status, kInvalidDecode, "unexpected end of file");
        m = d[pos++];
        seg = nullptr;
        len = 0;
        if (m == 0xD8 || m == 0xD9 || (m >= 0xD0 && m <= 0xD7)) return true;
        if (pos + 2 > n) return decode_fail(p.status, kInvalidDecode, "truncated marker");
        const size_t length = ((size_t)d[pos] << 8) | d[pos + 1];
        pos += 2;
        if (length < 2 || pos + length - 2 > n) return decode_fail(p.status, kInvalidDecode, "invalid marker length");
        seg = d + pos;
        len = length - 2;
        pos += length - 2;
        return true;
    }

    bool sof0(const uint8_t *s, size_t len)   // :294-357
    {
        if (len < 8) return decode_fail(p.status, kInvalidDecode, "invalid SOF0 length");
        if (s[0] != 8) return decode_fail(p.status, kUnsupportedDecode, "%u-bit precision not supported", s[0]);
        p.height = ((uint32_t)s[1] << 8) | s[2];
        p.width = ((uint32_t)s[3] << 8) | s[4];
        const uint32_t nc = s[5];
        if (nc != 1 && nc != 3) return decode_fail(p.status, kUnsupportedDecode, "%u components not supported", nc);
        if (len < 6 + nc * 3) return decode_fail(p.status, kInvalidDecode, "truncated SOF0 components");
        p.ncomp = 0;
        for (uint32_t i = 0; i < nc; ++i) {
            const uint8_t *c = s + 6 + i * 3;
            const uint8_t h = c[1] >> 4, v = c[1] & 15;
            if (h == 0 || v == 0)
                return decode_fail(p.status, kInvalidDecode, "invalid sampling factors %ux%u for component %u", h, v,
                                   c[0]);
            if (c[2] > 3)
                return decode_fail(p.status, kInvalidDecode, "invalid quantization table ID %u for component %u", c[2],
                                   c[0]);
            // the maxima are never reset: a second SOF0 keeps the first one's (:344-345)
            p.max_h = std::max<uint32_t>(p.max_h, h);
            p.max_v = std::max<uint32_t>(p.max_v, v);
            p.h[i] = h;
            p.v[i] = v;
            p.q[i] = c[2];
            p.dc[i] = p.ac[i] = 0;
            p.ncomp = i + 1;
        }
        return true;
    }

    bool dht(const uint8_t *s, size_t len)   // :359-396
    {
        size_t off = 0;
        while (off < len) {
            const uint8_t info = s[off];
            const uint32_t cls = info >> 4, id = info & 15;
            if (id > 3) return decode_fail(p.status, kInvalidDecode, "invalid Huffman table ID");
            ++off;
            if (off + 16 > len) return decode_fail(p.status, kInvalidDecode, "truncated DHT");
            const uint8_t *bits = s + off;
            off += 16;
            uint32_t nv = 0;
            for (int i = 0; i < 16; ++i) nv += bits[i];
            if (off + nv > len) return decode_fail(p.status, kInvalidDecode, "truncated DHT values");
            const int t = cls == 0 ? (int)id : 4 + (int)id;
            build_huff(bits, s + off, nv, p.tab[t], p.vals[t]);
            off += nv;
        }
        return true;
    }

    bool dqt(const uint8_t *s, size_t len)   // :398-434
    {
        size_t off = 0;
        while (off < len) {
            const uint8_t info = s[off];
            const uint32_t prec = info >> 4, id = info & 15;
            if (id > 3) return decode_fail(p.status, kInvalidDecode, "invalid quantization table ID");
            ++off;
            if (prec == 0) {
                if (off + 64 > len) return decode_fail(p.status, kInvalidDecode, "truncated DQT");
                for (int i = 0; i < 64; ++i) p.quant[id][i] = s[off + i];
                off += 64;
            } else {
                if (off + 128 > len) return decode_fail(p.status, kInvalidDecode, "truncated DQT");
                for (int i = 0; i < 64; ++i) p.quant[id][i] = (uint16_t)((s[off + 2 * i] << 8) | s[off + 2 * i + 1]);
                off += 128;
            }
        }
        return true;
    }

    bool sos(const uint8_t *s, size_t len)   // :446-484
    {
        if (len == 0) return decode_fail(p.status, kInvalidDecode, "empty SOS segment");
        if (s[0] != p.ncomp) return decode_fail(p.status, kInvalidDecode, "SOS component count mismatch");
        for (uint32_t i = 0; i < p.ncomp; ++i) {
            const size_t off = 1 + i * 2;
            if (off + 1 >= len) return decode_fail(p.status, kInvalidDecode, "truncated SOS segment");
            const uint8_t id = s[off], dc = s[off + 1] >> 4, ac = s[off + 1] & 15;
            if (dc > 3)
                return decode_fail(p.status, kInvalidDecode, "invalid DC Huffman table ID %u for component %u", dc, id);
            if (ac > 3)
                return decode_fail(p.status, kInvalidDecode, "invalid AC Huffman table ID %u for component %u", ac, id);
            p.dc[i] = dc;
            p.ac[i] = ac;
        }
        // an SOS with no components before any SOF0 passes pixo's checks and then panics in ycbcr_to_rgb
        // (components[1], :701); it is refused here instead
        if (p.ncomp == 0) return decode_fail(p.status, kInvalidDecode, "SOS with no frame components");
        return true;
    }

    // decode (:214-251)
    bool run()
    {
        if (n < 2 || d[0] != 0xFF || d[1] != 0xD8) return decode_fail(p.status, kInvalidDecode, "not a JPEG file");
        for (;;) {
            uint8_t m;
            const uint8_t *s;
            size_t len;
            if (!marker(m, s, len)) return false;
            bool ok = true;
            switch (m) {
            case 0xC0: ok = sof0(s, len); break;
            case 0xC2: return decode_fail(p.status, kUnsupportedDecode, "progressive JPEG not supported");
            case 0xC4: ok = dht(s, len); break;
            case 0xDB: ok = dqt(s, len); break;
            case 0xDD:   // parse_dri (:436-444)
                if (len != 2) return decode_fail(p.status, kInvalidDecode, "invalid DRI length");
                p.restart = ((uint32_t)s[0] << 8) | s[1];
                break;
            case 0xDA: return sos(s, len);
            case 0xD9: return decode_fail(p.status, kInvalidDecode, "no image data found");
            default: break;   // APPn, COM and unknown markers are skipped
            }
            if (!ok) return false;
        }
    }
};

}  // namespace

void parse(const uint8_t *data, size_t len, JdecParsed &p)
{
    p = JdecParsed();
    for (auto &t : p.tab) empty_huff(t);
    Parser P{data, len, 2, p};
    if (!P.run()) return;
    p.entropy = P.pos;
    p.entropy_len = jdec_entropy_end(data + P.pos, len - P.pos);
    p.out_ct = p.ncomp == 1 ? PIXO_B200_GRAY : PIXO_B200_RGB;
}

}  // namespace pixo
