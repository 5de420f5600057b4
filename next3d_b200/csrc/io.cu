// Host-side input parsers (SURVEY.md section 8 row f3): the per-frame FLAME mesh (.obj text) and landmark (.txt) files the
// inference scripts re-parse in Python for every frame (gen_samples_next3d.py:165-174, reenact_avatar_next3d.py:128-141,
// gen_videos_next3d.py:118-131).  Plain C++ (no device code): one pass over the text, strtod per number, so that the
// float64 -> float32 values are bit-identical to `float(token)` / `np.loadtxt` followed by `.float()`.
#include "common.cuh"
#include <stdlib.h>
#include <string.h>
#include <charconv>

namespace {

// str.split() separators (ASCII subset)
inline bool is_space(char c) { return c == ' ' || c == '\t' || c == '\n' || c == '\r' || c == '\v' || c == '\f'; }

// One token -> double with Python float() semantics for the spellings that occur in mesh files: correctly rounded decimal /
// exponent notation (std::from_chars, no locale, no allocation), optional leading '+', inf / nan; anything else (or trailing
// garbage) is an error, as float() raises.
bool parse_double(const char* p, const char* q, double& v) {
    if (p < q && *p == '+') {
        ++p;
        if (p < q && (*p == '+' || *p == '-')) return false;
    }
    const std::from_chars_result r = std::from_chars(p, q, v, std::chars_format::general);
    if (r.ec == std::errc::result_out_of_range) {           // from_chars leaves v untouched: fall back to strtod's +-inf / 0 / denormal
        char buf[128];
        const size_t len = (size_t)(q - p);
        if (len >= sizeof(buf)) return false;
        memcpy(buf, p, len);
        buf[len] = 0;
        char* stop = nullptr;
        v = strtod(buf, &stop);
        return stop == buf + len;
    }
    return r.ec == std::errc() && r.ptr == q;
}

// Parse the whitespace-separated numbers of [p, end) into out[n...]; returns false on a token that is not a number.
bool parse_numbers(const char* p, const char* end, float* out, int64_t cap, int64_t& n, int64_t& count_in_line) {
    count_in_line = 0;
    while (p < end) {
        while (p < end && is_space(*p)) ++p;
        if (p >= end) break;
        const char* q = p;
        while (q < end && !is_space(*q)) ++q;
        double v;
        if (!parse_double(p, q, v)) return false;
        if (n < cap) out[n] = (float)v;                     // float64 -> float32, like torch's .float()
        ++n;
        ++count_in_line;
        p = q;
    }
    return true;
}

}  // namespace

extern "C" int n3d_parse_obj_vertices(const char* text, int64_t len, float* xyz, int64_t max_vertices, int64_t* n_vertices) {
    N3D_CHECK_ARG(text && len >= 0 && n_vertices && (xyz || max_vertices == 0), "n3d_parse_obj_vertices: bad args");
    const char* p = text;
    const char* end = text + len;
    int64_t n = 0;
    while (p < end) {
        const char* eol = (const char*)memchr(p, '\n', (size_t)(end - p));
        const char* line_end = eol ? eol : end;
        if (line_end - p >= 2 && p[0] == 'v' && p[1] == ' ') {                 // `line[:2] == "v "`: not vt / vn / vp
            int64_t in_line = 0;
            if (!parse_numbers(p + 2, line_end, xyz, max_vertices * 3, n, in_line)) {
                n3d_set_error("n3d_parse_obj_vertices: malformed number in a vertex line (byte offset %lld)", (long long)(p - text));
                return N3D_ERR_INVALID_ARG;
            }
        }
        p = eol ? eol + 1 : end;
    }
    // the reference flattens all numbers and reshapes to (-1, 3): a count that is not a multiple of 3 is an error there too
    N3D_CHECK_ARG(n % 3 == 0, "n3d_parse_obj_vertices: %lld coordinates are not a multiple of 3", (long long)n);
    *n_vertices = n / 3;
    if (n / 3 > max_vertices) {
        n3d_set_error("n3d_parse_obj_vertices: %lld vertices, room for %lld", (long long)(n / 3), (long long)max_vertices);
        return N3D_ERR_INVALID_ARG;
    }
    return N3D_OK;
}

extern "C" int n3d_parse_float_table(const char* text, int64_t len, float* values, int64_t max_values, int64_t* n_values, int64_t* n_cols) {
    N3D_CHECK_ARG(text && len >= 0 && n_values && n_cols && (values || max_values == 0), "n3d_parse_float_table: bad args");
    const char* p = text;
    const char* end = text + len;
    int64_t n = 0, cols = -1;
    while (p < end) {
        const char* eol = (const char*)memchr(p, '\n', (size_t)(end - p));
        const char* line_end = eol ? eol : end;
        const char* hash = (const char*)memchr(p, '#', (size_t)(line_end - p));   // np.loadtxt: '#' starts a comment
        int64_t in_line = 0;
        if (!parse_numbers(p, hash ? hash : line_end, values, max_values, n, in_line)) {
            n3d_set_error("n3d_parse_float_table: malformed number (byte offset %lld)", (long long)(p - text));
            return N3D_ERR_INVALID_ARG;
        }
        if (in_line > 0) {                                                       // blank / comment-only lines are skipped
            if (cols < 0) cols = in_line;
            N3D_CHECK_ARG(in_line == cols, "n3d_parse_float_table: a row has %lld columns, the first one %lld", (long long)in_line, (long long)cols);
        }
        p = eol ? eol + 1 : end;
    }
    *n_values = n;
    *n_cols = cols < 0 ? 0 : cols;
    if (n > max_values) {
        n3d_set_error("n3d_parse_float_table: %lld values, room for %lld", (long long)n, (long long)max_values);
        return N3D_ERR_INVALID_ARG;
    }
    return N3D_OK;
}
