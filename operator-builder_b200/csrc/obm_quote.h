/*
 * obm_quote.h -- strconv.Quote (what fmt's %q prints for a string) of Go 1.16, host only.  The lexer's messages
 * (error.go:18,40, state.go:193,259,270 through obm_decode.cpp) and the parser's strconv / unmarshal / missing-argument
 * messages (obm_parse.cpp) quote with it.
 *
 * Rune by rune (quote.go appendQuotedWith / appendEscapedRune): an invalid byte prints as \xHH; '"' and '\\' are
 * escaped; a strconv.IsPrint rune (Unicode 13.0, GO_PRINT_RANGES) is copied; \a \b \f \n \r \t \v by name; any other
 * rune below U+0020 as \xHH, the rest as \uHHHH or \UHHHHHHHH -- DEL included (\u007f: Go 1.16 has no \x7f case).
 */
#ifndef OBM_QUOTE_H
#define OBM_QUOTE_H

#include <cstdint>
#include <string>

#include "go_unicode_tables.h"
#include "obm_core.h"

namespace obm {

inline bool go_is_print(int r) { return r >= 0 && in_ranges(GO_PRINT_RANGES, GO_PRINT_RANGES_N, r); }

inline void go_quote(std::string &out, const std::string &s) {
    static const char hex[] = "0123456789abcdef";
    const uint8_t *b = (const uint8_t *)s.data();
    const uint32_t n = (uint32_t)s.size();
    out.push_back('"');
    uint32_t i = 0;
    while (i < n) {
        uint32_t w = 1; int r = b[i];
        if (r >= 0x80) r = decode_rune(b, i, n, w);
        if (w == 1 && r == RUNE_ERR) { out += "\\x"; out.push_back(hex[b[i] >> 4]); out.push_back(hex[b[i] & 0xF]); i += 1; continue; }
        if (r == '"' || r == '\\') { out.push_back('\\'); out.push_back((char)r); i += w; continue; }
        if (go_is_print(r)) { out.append((const char *)b + i, w); i += w; continue; }
        switch (r) {
        case '\a': out += "\\a"; break;
        case '\b': out += "\\b"; break;
        case '\f': out += "\\f"; break;
        case '\n': out += "\\n"; break;
        case '\r': out += "\\r"; break;
        case '\t': out += "\\t"; break;
        case '\v': out += "\\v"; break;
        default:
            if (r < ' ') { out += "\\x"; out.push_back(hex[(r >> 4) & 0xF]); out.push_back(hex[r & 0xF]); }
            else if (r < 0x10000) { out += "\\u"; for (int sh = 12; sh >= 0; sh -= 4) out.push_back(hex[(r >> sh) & 0xF]); }
            else { out += "\\U"; for (int sh = 28; sh >= 0; sh -= 4) out.push_back(hex[(r >> sh) & 0xF]); }
        }
        i += w;
    }
    out.push_back('"');
}

inline std::string go_quote(const std::string &s) { std::string o; go_quote(o, s); return o; }

} // namespace obm

#endif
