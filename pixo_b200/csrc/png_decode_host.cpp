// png_decode_host.cpp — the host half of the PNG decoder: the chunk walk, the checks after it and the zlib header,
// as pixo::decode::decode_png makes them (src/decode/png.rs:101-263, src/decode/inflate.rs:294-320).  Chunk headers
// are a few bytes each, so they are walked here; the IDAT CRCs, inflate, unfiltering and expansion run on the device
// (png_decode.cu).
#include "png_decode_host.hpp"

#include <string.h>

namespace pixo {

namespace {

struct CrcTable {
    uint32_t t[256];
    CrcTable()
    {
        for (uint32_t i = 0; i < 256; ++i) {
            uint32_t c = i;
            for (int k = 0; k < 8; ++k) c = c & 1 ? (c >> 1) ^ 0xEDB88320u : c >> 1;
            t[i] = c;
        }
    }
};
const CrcTable kCrc;

uint32_t be32(const uint8_t *p) { return (uint32_t)p[0] << 24 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 8 | p[3]; }

// String::from_utf8_lossy of a chunk type: each maximal invalid prefix of a sequence becomes U+FFFD
std::string utf8_lossy(const uint8_t *s, size_t n)
{
    std::string out;
    for (size_t i = 0; i < n;) {
        const uint8_t b = s[i];
        size_t need = 0;
        uint8_t lo = 0x80, hi = 0xBF;
        if (b < 0x80) {
            out += (char)b;
            ++i;
            continue;
        } else if (b >= 0xC2 && b <= 0xDF) {
            need = 1;
        } else if (b >= 0xE0 && b <= 0xEF) {
            need = 2;
            if (b == 0xE0) lo = 0xA0;
            if (b == 0xED) hi = 0x9F;
        } else if (b >= 0xF0 && b <= 0xF4) {
            need = 3;
            if (b == 0xF0) lo = 0x90;
            if (b == 0xF4) hi = 0x8F;
        }
        size_t k = 1;
        bool ok = need > 0;
        for (; ok && k <= need; ++k) {
            if (i + k >= n) { ok = false; break; }
            const uint8_t c = s[i + k];
            if (c < (k == 1 ? lo : 0x80) || c > (k == 1 ? hi : 0xBF)) { ok = false; break; }
        }
        if (ok) {
            out.append(reinterpret_cast<const char *>(s + i), need + 1);
            i += need + 1;
        } else {
            out += "\xEF\xBF\xBD";
            i += need > 0 ? k : 1;
        }
    }
    return out;
}

const char *ctype_name(uint8_t c)
{
    switch (c) {
    case 0: return "Grayscale";
    case 2: return "Rgb";
    case 3: return "Indexed";
    case 4: return "GrayscaleAlpha";
    default: return "Rgba";
    }
}

}  // namespace

uint32_t crc32_update(uint32_t reg, const uint8_t *p, size_t n)
{
    for (size_t i = 0; i < n; ++i) reg = (reg >> 8) ^ kCrc.t[(reg ^ p[i]) & 0xFF];
    return reg;
}

// The walk and the checks after it, false for a file refused; with check_idat_crc the IDAT CRCs are checked as well
static bool walk(const uint8_t *data, size_t len, PdecParsed &p, bool check_idat_crc)
{
    p = PdecParsed();
    static const uint8_t kSig[8] = {0x89, 0x50, 0x4E, 0x47, 0x0D, 0x0A, 0x1A, 0x0A};
    if (len < 8 || memcmp(data, kSig, 8) != 0) return decode_fail(p.status, kInvalidDecode, "not a PNG file");
    bool have_ihdr = false, seen_iend = false;
    uint8_t comp = 0, filt = 0, interlace = 0;
    size_t pos = 8;
    while (pos + 12 <= len) {
        const uint64_t length = be32(data + pos);
        const uint8_t *type = data + pos + 4;
        const uint64_t start = pos + 8, end = start + length, crc_end = end + 4;
        if (crc_end > len) return decode_fail(p.status, kInvalidDecode, "truncated PNG chunk");
        const uint8_t *d = data + start;
        const uint32_t stored = be32(data + end);
        const bool idat = memcmp(type, "IDAT", 4) == 0;
        if (!idat || check_idat_crc) {
            const uint32_t crc = crc32_update(crc32_update(0xFFFFFFFFu, type, 4), d, length) ^ 0xFFFFFFFFu;
            if (crc != stored)
                return decode_fail(p.status, kInvalidDecode, "CRC mismatch in %s chunk", utf8_lossy(type, 4).c_str());
        }
        if (memcmp(type, "IHDR", 4) == 0) {
            if (length != 13) return decode_fail(p.status, kInvalidDecode, "invalid IHDR length");
            const uint8_t ct = d[9];
            if (ct != 0 && ct != 2 && ct != 3 && ct != 4 && ct != 6)
                return decode_fail(p.status, kInvalidDecode, "invalid PNG color type: %u", ct);
            have_ihdr = true;
            p.width = be32(d);
            p.height = be32(d + 4);
            p.depth = d[8];
            p.ctype = ct;
            comp = d[10];
            filt = d[11];
            interlace = d[12];
        } else if (memcmp(type, "PLTE", 4) == 0) {
            if (length % 3 != 0) return decode_fail(p.status, kInvalidDecode, "invalid PLTE length");
            p.has_plte = true;
            p.plte.assign(d, d + length);
        } else if (memcmp(type, "tRNS", 4) == 0) {
            p.trns.assign(d, d + length);
        } else if (idat) {
            p.idat_off.push_back(start);
            p.idat_len.push_back((uint32_t)length);
            p.idat_crc.push_back(stored);
            p.idat_total += length;
        } else if (memcmp(type, "IEND", 4) == 0) {
            seen_iend = true;
            break;
        }
        pos = crc_end;
    }
    if (!seen_iend) return decode_fail(p.status, kInvalidDecode, "missing IEND chunk");
    if (!have_ihdr) return decode_fail(p.status, kInvalidDecode, "missing IHDR chunk");
    if (p.width == 0 || p.height == 0)
        return decode_fail(p.status, PIXO_B200_ERR_INVALID_DIMENSIONS, "Invalid image dimensions: %ux%u", p.width,
                           p.height);
    if (p.width > (1u << 24) || p.height > (1u << 24))
        return decode_fail(p.status, PIXO_B200_ERR_IMAGE_TOO_LARGE, "Image %ux%u exceeds maximum dimension %u", p.width,
                           p.height, 1u << 24);
    if (comp != 0) return decode_fail(p.status, kInvalidDecode, "unsupported compression method");
    if (filt != 0) return decode_fail(p.status, kInvalidDecode, "unsupported filter method");
    if (interlace != 0) return decode_fail(p.status, kUnsupportedDecode, "Adam7 interlaced images not supported");
    const uint8_t bd = p.depth;
    bool ok;
    switch (p.ctype) {
    case 0: ok = bd == 1 || bd == 2 || bd == 4 || bd == 8 || bd == 16; break;
    case 3: ok = bd == 1 || bd == 2 || bd == 4 || bd == 8; break;
    default: ok = bd == 8 || bd == 16; break;
    }
    if (!ok)
        return decode_fail(p.status, kInvalidDecode, "invalid bit depth %u for color type %s", bd, ctype_name(p.ctype));
    if (p.idat_total == 0) return decode_fail(p.status, kInvalidDecode, "no IDAT data");
    const uint64_t w = p.width;
    static const uint32_t kChannels[7] = {1, 0, 3, 1, 2, 0, 4};
    const uint32_t ch = kChannels[p.ctype];
    if (p.ctype == 0 || p.ctype == 3) {
        p.sb = (w * bd + 7) / 8;
        p.bpp = bd == 16 ? 2 : 1;
    } else {
        p.bpp = ch * bd / 8;
        p.sb = w * p.bpp;
    }
    p.expected = (uint64_t)p.height * (1 + p.sb);
    // the zlib header: the IDAT payloads concatenated, as inflate_zlib_with_size sees them
    if (p.idat_total < 6) return decode_fail(p.status, kInvalidDecode, "zlib stream too short");
    uint8_t hdr[2];
    for (size_t c = 0, k = 0; c < p.idat_off.size() && k < 2; ++c)
        for (uint32_t j = 0; j < p.idat_len[c] && k < 2; ++j) hdr[k++] = data[p.idat_off[c] + j];
    if ((hdr[0] & 0x0F) != 8) return decode_fail(p.status, kInvalidDecode, "invalid zlib compression method");
    if ((((uint32_t)hdr[0] << 8) | hdr[1]) % 31 != 0)
        return decode_fail(p.status, kInvalidDecode, "invalid zlib header checksum");
    if (hdr[1] & 0x20) return decode_fail(p.status, kUnsupportedDecode, "preset dictionary not supported");
    // the frame decode_png returns
    bool alpha = false;
    for (uint8_t a : p.trns) alpha |= a != 0xFF;
    switch (p.ctype) {
    case 0: p.out_ct = PIXO_B200_GRAY; p.out_channels = 1; break;
    case 4: p.out_ct = PIXO_B200_GRAY_ALPHA; p.out_channels = 2; break;
    case 2: p.out_ct = PIXO_B200_RGB; p.out_channels = 3; break;
    case 6: p.out_ct = PIXO_B200_RGBA; p.out_channels = 4; break;
    default:
        p.out_ct = alpha ? PIXO_B200_RGBA : PIXO_B200_RGB;
        p.out_channels = alpha ? 4 : 3;
        break;
    }
    return true;
}

void parse(const uint8_t *data, size_t len, PdecParsed &p)
{
    if (!walk(data, len, p, false)) walk(data, len, p, true);
}

}  // namespace pixo
