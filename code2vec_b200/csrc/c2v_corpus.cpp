// c2v_corpus.cpp -- host side of the data path: the corpus reader and the code-vector writer either side of
// the hot path, in C++ behind the same C ABI (no torch, no Python in here).
//
//   c2v_corpus_parse_files   DatasetReader.load (/root/reference/model/dataset_reader.py:72-128): the `corpus.txt`
//                            text format -> CSR arrays (contexts int32 [n][3] with the @question shift already applied,
//                            offsets, ids, raw label / alias strings) that DeviceCorpus uploads as they are
//   c2v_corpus_save / _load  binary cache of the parsed corpus (one flat file; top11: 1.07 GB of text -> ~1 GB of int32)
//   c2v_write_code_vectors   write_code_vectors (/root/reference/main.py:393-423): `label\tv0 v1 ...` lines and the
//                            test-result TSV, every float printed exactly like Python's str(float) (shortest round
//                            trip of the double the fp32 value converts to)
//
// Line semantics reproduced from the reference parser: a line is stripped of ' \r\n\t' on both ends; an empty line
// closes the current item; any other line opens one; `#<id>`, `label:`, `class:`, `paths:`, `vars:`, `doc:` are tested
// in that order; the paths / vars mode is NOT reset between items (dataset_reader.py:76, :107-110); a context line is
// `start\tpath\tend` with start and end shifted by QUESTION_TOKEN_INDEX (:113-115); a vars line is
// `original\talias` (:117-119).  Label normalisation (Vocab.normalize_method_name + lower(), dataset.py:86-92) is
// done by the Python mirror on the UNIQUE strings only, because str.lower() is Unicode-aware.
#include <charconv>
#include <cerrno>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include "../../include/c2v_b200.h"

namespace c2v {
void set_error(const char *fmt, ...);
}
using c2v::set_error;

struct c2v_corpus {
    std::vector<int64_t> ids;             // [n_items]  (-1: the item had no '#' line; the reference keeps None)
    std::vector<int64_t> ctx_off;         // [n_items + 1]
    std::vector<int32_t> ctx;             // [n_contexts][3]
    std::vector<int64_t> label_off;       // [n_items + 1] into label_blob (raw text after "label:")
    std::string label_blob;
    std::vector<uint8_t> has_label;       // [n_items]
    std::vector<int32_t> label_pos;       // [n_items] aliases of the item parsed BEFORE its label: line (vocab insertion order)
    std::vector<int64_t> alias_item_off;  // [n_items + 1] into the alias arrays
    std::vector<int64_t> alias_orig_off;  // [n_aliases + 1] into alias_blob: original variable name
    std::vector<int64_t> alias_name_off;  // [n_aliases + 1] into alias_name_blob: alias (@var_k, ...)
    std::string alias_blob, alias_name_blob;
};

namespace {

inline bool is_strip(char c) { return c == ' ' || c == '\r' || c == '\n' || c == '\t'; }

// Python int() of a field of a context line: optional surrounding whitespace, optional sign, decimal digits
// (underscores between digits are legal in Python; the corpus never has them and they are rejected here)
bool parse_int(const char *b, const char *e, long long *out)
{
    while (b < e && (is_strip(*b) || *b == '\f' || *b == '\v')) ++b;
    while (e > b && (is_strip(e[-1]) || e[-1] == '\f' || e[-1] == '\v')) --e;
    if (b == e) return false;
    bool neg = false;
    if (*b == '+' || *b == '-') { neg = *b == '-'; ++b; }
    if (b == e) return false;
    long long v = 0;
    for (; b < e; ++b) {
        if (*b < '0' || *b > '9') return false;
        if (v > (INT64_MAX - 9) / 10) return false;
        v = v * 10 + (*b - '0');
    }
    *out = neg ? -v : v;
    return true;
}

struct Parser {
    c2v_corpus *c;
    int shift;
    int mode = 0;            // 0: none, 1: paths, 2: vars  (persists across items like the reference's parse_mode)
    bool open = false;       // an item is being filled
    long long line_no = 0;
    std::string err;

    void open_item()
    {
        c->ids.push_back(-1);
        c->has_label.push_back(0);
        c->label_pos.push_back(0);
        open = true;
    }
    void close_item()
    {
        if (!open) return;
        c->ctx_off.push_back((int64_t)(c->ctx.size() / 3));
        c->label_off.push_back((int64_t)c->label_blob.size());
        c->alias_item_off.push_back((int64_t)(c->alias_orig_off.size() - 1));
        open = false;
    }
    bool fail(const char *what, const char *b, const char *e)
    {
        char buf[256];
        snprintf(buf, sizeof(buf), "corpus line %lld: %s: '%.*s'", line_no, what, (int)((e - b) > 80 ? 80 : (e - b)), b);
        err = buf;
        return false;
    }
    // one raw line (without its terminator)
    bool line(const char *b, const char *e)
    {
        ++line_no;
        while (b < e && is_strip(*b)) ++b;
        while (e > b && is_strip(e[-1])) --e;
        if (b == e) { close_item(); return true; }
        if (!open) open_item();
        const size_t n = (size_t)(e - b);
        if (*b == '#') {
            long long v;
            if (!parse_int(b + 1, e, &v)) return fail("invalid literal for int()", b, e);
            c->ids.back() = v;
        } else if (n >= 6 && !memcmp(b, "label:", 6)) {
            // The reference appends to the label vocabulary at every label: line (:99-100); an item with two of them
            // would need both, in order.  No corpus the preprocessor writes has that: refuse instead of guessing.
            if (c->has_label.back()) return fail("second label: line in one item (not supported)", b, e);
            c->label_blob.append(b + 6, e);
            c->has_label.back() = 1;
            c->label_pos.back() = (int32_t)((int64_t)(c->alias_orig_off.size() - 1) - c->alias_item_off.back());
        } else if (n >= 6 && !memcmp(b, "class:", 6)) {
            // CodeData.source: never read by the training / export path
        } else if (n >= 6 && !memcmp(b, "paths:", 6)) {
            mode = 1;
        } else if (n >= 5 && !memcmp(b, "vars:", 5)) {
            mode = 2;
        } else if (n >= 4 && !memcmp(b, "doc:", 4)) {
        } else if (mode == 1) {
            const char *f[3]; const char *g[3];
            const char *p = b;
            for (int k = 0; k < 3; ++k) {
                if (p > e) return fail("list index out of range (context line needs 3 tab-separated fields)", b, e);
                const char *t = (const char *)memchr(p, '\t', (size_t)(e - p));
                f[k] = p; g[k] = t ? t : e;
                p = t ? t + 1 : e + 1;
            }
            long long v[3];
            for (int k = 0; k < 3; ++k)
                if (!parse_int(f[k], g[k], &v[k])) return fail("invalid literal for int()", b, e);
            v[0] += shift; v[2] += shift;
            for (int k = 0; k < 3; ++k)
                if (v[k] < INT32_MIN || v[k] > INT32_MAX) return fail("index does not fit 32 bits", b, e);
            c->ctx.push_back((int32_t)v[0]); c->ctx.push_back((int32_t)v[1]); c->ctx.push_back((int32_t)v[2]);
        } else if (mode == 2) {
            const char *t = (const char *)memchr(b, '\t', n);
            if (!t) return fail("list index out of range (vars line needs original<TAB>alias)", b, e);
            const char *a0 = t + 1;
            const char *t2 = (const char *)memchr(a0, '\t', (size_t)(e - a0));
            const char *a1 = t2 ? t2 : e;
            c->alias_blob.append(b, t);
            c->alias_orig_off.push_back((int64_t)c->alias_blob.size());
            c->alias_name_blob.append(a0, a1);
            c->alias_name_off.push_back((int64_t)c->alias_name_blob.size());
        }
        return true;
    }
};

// feeds a byte stream to the parser line by line with Python's universal-newline rules ('\n', '\r\n' and a lone '\r'
// all end a line); `carry` holds an unterminated tail across chunk (file) boundaries, `pending_cr` a '\r' that ended a chunk
struct LineFeeder {
    Parser *p;
    std::string carry;
    bool pending_cr = false;
    bool feed(const char *b, size_t n)
    {
        const char *e = b + n;
        if (pending_cr) { pending_cr = false; if (b < e && *b == '\n') ++b; }
        while (b < e) {
            const char *q = b;
            while (q < e && *q != '\n' && *q != '\r') ++q;      // (memchr2 by hand: lines are short)
            if (q == e) { carry.append(b, e); return true; }
            bool ok;
            if (!carry.empty()) { carry.append(b, q); ok = p->line(carry.data(), carry.data() + carry.size()); carry.clear(); }
            else ok = p->line(b, q);
            if (!ok) return false;
            if (*q == '\r') {
                if (q + 1 < e) { b = (q[1] == '\n') ? q + 2 : q + 1; }
                else { pending_cr = true; b = q + 1; }
            } else b = q + 1;
        }
        return true;
    }
    bool finish()
    {
        if (!carry.empty()) { if (!p->line(carry.data(), carry.data() + carry.size())) return false; carry.clear(); }
        p->close_item();                                        // dataset_reader.py:127-128
        return true;
    }
};

c2v_corpus *new_corpus()
{
    c2v_corpus *c = new c2v_corpus();
    c->ctx_off.push_back(0); c->label_off.push_back(0); c->alias_item_off.push_back(0);
    c->alias_orig_off.push_back(0); c->alias_name_off.push_back(0);
    return c;
}

// Python's repr(float) ("short" float_repr_style): the shortest digit string that round-trips, fixed notation for
// -4 < decimal exponent <= 16, scientific otherwise ("1e-05", "1.5e+16"), always with a '.0' or an exponent.
size_t py_float_repr(double x, char *out)
{
    if (x != x) { memcpy(out, "nan", 3); return 3; }
    char *o = out;
    if (x == 0.0) { if (std::signbit(x)) *o++ = '-'; memcpy(o, "0.0", 3); return (size_t)(o + 3 - out); }
    if (x < 0) { *o++ = '-'; x = -x; }
    if (x > 1.7976931348623157e308) { memcpy(o, "inf", 3); return (size_t)(o + 3 - out); }
    char sci[40];
    auto r = std::to_chars(sci, sci + sizeof(sci), x, std::chars_format::scientific);   // d[.ddd]e[+-]XX, shortest
    const char *epos = (const char *)memchr(sci, 'e', (size_t)(r.ptr - sci));
    char digits[24]; int nd = 0;
    for (const char *q = sci; q < epos; ++q) if (*q != '.') digits[nd++] = *q;
    int ex = 0;
    std::from_chars(epos + (epos[1] == '+' ? 2 : 1), r.ptr, ex);
    const int decpt = ex + 1;                                   // value = 0.d1d2... x 10^decpt
    if (decpt <= -4 || decpt > 16) {
        *o++ = digits[0];
        if (nd > 1) { *o++ = '.'; memcpy(o, digits + 1, (size_t)nd - 1); o += nd - 1; }
        *o++ = 'e';
        int e10 = decpt - 1;
        *o++ = e10 < 0 ? '-' : '+';
        if (e10 < 0) e10 = -e10;
        char eb[8]; int ne = 0;
        do { eb[ne++] = (char)('0' + e10 % 10); e10 /= 10; } while (e10);
        if (ne < 2) eb[ne++] = '0';
        while (ne) *o++ = eb[--ne];
    } else if (decpt <= 0) {
        *o++ = '0'; *o++ = '.';
        for (int i = 0; i < -decpt; ++i) *o++ = '0';
        memcpy(o, digits, (size_t)nd); o += nd;
    } else if (decpt >= nd) {
        memcpy(o, digits, (size_t)nd); o += nd;
        for (int i = 0; i < decpt - nd; ++i) *o++ = '0';
        *o++ = '.'; *o++ = '0';
    } else {
        memcpy(o, digits, (size_t)decpt); o += decpt;
        *o++ = '.';
        memcpy(o, digits + decpt, (size_t)(nd - decpt)); o += nd - decpt;
    }
    return (size_t)(o - out);
}

const uint64_t kCacheMagic = 0x3176707263763263ull;             // "c2vcrpv1"

template <typename T>
bool put_vec(FILE *f, const std::vector<T> &v)
{
    const uint64_t n = v.size();
    return fwrite(&n, 8, 1, f) == 1 && (n == 0 || fwrite(v.data(), sizeof(T), n, f) == n);
}
bool put_str(FILE *f, const std::string &s)
{
    const uint64_t n = s.size();
    return fwrite(&n, 8, 1, f) == 1 && (n == 0 || fwrite(s.data(), 1, n, f) == n);
}
template <typename T>
bool get_vec(FILE *f, std::vector<T> &v)
{
    uint64_t n = 0;
    if (fread(&n, 8, 1, f) != 1 || n > (1ull << 40)) return false;
    v.resize(n);
    return n == 0 || fread(v.data(), sizeof(T), n, f) == n;
}
bool get_str(FILE *f, std::string &s)
{
    uint64_t n = 0;
    if (fread(&n, 8, 1, f) != 1 || n > (1ull << 40)) return false;
    s.resize(n);
    return n == 0 || fread(&s[0], 1, n, f) == n;
}

}  // namespace

extern "C" {

int c2v_corpus_parse_buffer(const char *text, size_t n, int32_t question_shift, c2v_corpus **out)
{
    if (!out || (!text && n)) { set_error("c2v_corpus_parse_buffer: NULL argument"); return C2V_EINVAL; }
    c2v_corpus *c = new_corpus();
    Parser p; p.c = c; p.shift = question_shift;
    LineFeeder lf; lf.p = &p;
    if (!lf.feed(text, n) || !lf.finish()) { set_error("%s", p.err.c_str()); delete c; return C2V_EINVAL; }
    *out = c;
    return C2V_OK;
}

int c2v_corpus_parse_files(const char *const *paths, int32_t n_paths, int32_t question_shift, c2v_corpus **out)
{
    if (!out || !paths || n_paths < 1) { set_error("c2v_corpus_parse_files: bad argument"); return C2V_EINVAL; }
    c2v_corpus *c = new_corpus();
    Parser p; p.c = c; p.shift = question_shift;
    LineFeeder lf; lf.p = &p;
    for (int i = 0; i < n_paths; ++i) {                        // the files are read as one concatenated stream (`cat`)
        const int fd = open(paths[i], O_RDONLY);
        if (fd < 0) { set_error("cannot open %s: %s", paths[i], strerror(errno)); delete c; return C2V_EINVAL; }
        struct stat st;
        if (fstat(fd, &st) != 0) { set_error("fstat %s: %s", paths[i], strerror(errno)); close(fd); delete c; return C2V_EINVAL; }
        if (st.st_size > 0) {
            void *m = mmap(nullptr, (size_t)st.st_size, PROT_READ, MAP_PRIVATE, fd, 0);
            if (m == MAP_FAILED) { set_error("mmap %s: %s", paths[i], strerror(errno)); close(fd); delete c; return C2V_EINVAL; }
            madvise(m, (size_t)st.st_size, MADV_SEQUENTIAL);
            const bool ok = lf.feed((const char *)m, (size_t)st.st_size);
            munmap(m, (size_t)st.st_size);
            if (!ok) { set_error("%s: %s", paths[i], p.err.c_str()); close(fd); delete c; return C2V_EINVAL; }
        }
        close(fd);
    }
    if (!lf.finish()) { set_error("%s", p.err.c_str()); delete c; return C2V_EINVAL; }
    *out = c;
    return C2V_OK;
}

void c2v_corpus_free(c2v_corpus *c) { delete c; }

int c2v_corpus_get_info(const c2v_corpus *c, c2v_corpus_info *info)
{
    if (!c || !info) { set_error("c2v_corpus_get_info: NULL argument"); return C2V_EINVAL; }
    info->n_items = (int64_t)c->ids.size();
    info->n_contexts = (int64_t)(c->ctx.size() / 3);
    info->n_aliases = (int64_t)(c->alias_orig_off.size() - 1);
    info->label_bytes = (int64_t)c->label_blob.size();
    info->alias_bytes = (int64_t)c->alias_blob.size();
    info->alias_name_bytes = (int64_t)c->alias_name_blob.size();
    return C2V_OK;
}

int c2v_corpus_export(const c2v_corpus *c, int64_t *ids, int64_t *ctx_offsets, int32_t *contexts,
                      int64_t *label_offsets, char *label_blob, uint8_t *has_label, int32_t *label_pos,
                      int64_t *alias_item_offsets,
                      int64_t *alias_orig_offsets, char *alias_blob, int64_t *alias_name_offsets, char *alias_name_blob)
{
    if (!c) { set_error("c2v_corpus_export: NULL corpus"); return C2V_EINVAL; }
    auto cp = [](void *dst, const void *src, size_t n) { if (dst && n) memcpy(dst, src, n); };
    cp(ids, c->ids.data(), c->ids.size() * 8);
    cp(ctx_offsets, c->ctx_off.data(), c->ctx_off.size() * 8);
    cp(contexts, c->ctx.data(), c->ctx.size() * 4);
    cp(label_offsets, c->label_off.data(), c->label_off.size() * 8);
    cp(label_blob, c->label_blob.data(), c->label_blob.size());
    cp(has_label, c->has_label.data(), c->has_label.size());
    cp(label_pos, c->label_pos.data(), c->label_pos.size() * 4);
    cp(alias_item_offsets, c->alias_item_off.data(), c->alias_item_off.size() * 8);
    cp(alias_orig_offsets, c->alias_orig_off.data(), c->alias_orig_off.size() * 8);
    cp(alias_blob, c->alias_blob.data(), c->alias_blob.size());
    cp(alias_name_offsets, c->alias_name_off.data(), c->alias_name_off.size() * 8);
    cp(alias_name_blob, c->alias_name_blob.data(), c->alias_name_blob.size());
    return C2V_OK;
}

int c2v_corpus_save(const c2v_corpus *c, const char *path)
{
    if (!c || !path) { set_error("c2v_corpus_save: NULL argument"); return C2V_EINVAL; }
    FILE *f = fopen(path, "wb");
    if (!f) { set_error("cannot open %s: %s", path, strerror(errno)); return C2V_EINVAL; }
    bool ok = fwrite(&kCacheMagic, 8, 1, f) == 1 && put_vec(f, c->ids) && put_vec(f, c->ctx_off) && put_vec(f, c->ctx) &&
              put_vec(f, c->label_off) && put_str(f, c->label_blob) && put_vec(f, c->has_label) && put_vec(f, c->label_pos) &&
              put_vec(f, c->alias_item_off) && put_vec(f, c->alias_orig_off) && put_str(f, c->alias_blob) &&
              put_vec(f, c->alias_name_off) && put_str(f, c->alias_name_blob);
    ok = (fclose(f) == 0) && ok;
    if (!ok) { set_error("short write to %s", path); return C2V_EINVAL; }
    return C2V_OK;
}

int c2v_corpus_load(const char *path, c2v_corpus **out)
{
    if (!out || !path) { set_error("c2v_corpus_load: NULL argument"); return C2V_EINVAL; }
    FILE *f = fopen(path, "rb");
    if (!f) { set_error("cannot open %s: %s", path, strerror(errno)); return C2V_EINVAL; }
    c2v_corpus *c = new c2v_corpus();
    uint64_t magic = 0;
    bool ok = fread(&magic, 8, 1, f) == 1 && magic == kCacheMagic && get_vec(f, c->ids) && get_vec(f, c->ctx_off) &&
              get_vec(f, c->ctx) && get_vec(f, c->label_off) && get_str(f, c->label_blob) && get_vec(f, c->has_label) && get_vec(f, c->label_pos) &&
              get_vec(f, c->alias_item_off) && get_vec(f, c->alias_orig_off) && get_str(f, c->alias_blob) &&
              get_vec(f, c->alias_name_off) && get_str(f, c->alias_name_blob);
    fclose(f);
    const size_t n = c->ids.size();
    ok = ok && c->ctx_off.size() == n + 1 && c->label_off.size() == n + 1 && c->has_label.size() == n && c->label_pos.size() == n &&
         c->alias_item_off.size() == n + 1 && c->ctx.size() == (size_t)c->ctx_off.back() * 3 &&
         c->alias_orig_off.size() == c->alias_name_off.size() && !c->alias_orig_off.empty() &&
         (size_t)c->alias_item_off.back() == c->alias_orig_off.size() - 1 &&
         (size_t)c->label_off.back() == c->label_blob.size();
    if (!ok) { set_error("%s is not a c2v corpus cache (or is truncated)", path); delete c; return C2V_EINVAL; }
    *out = c;
    return C2V_OK;
}

int c2v_format_float(float value, char *out, size_t out_bytes)
{
    char buf[48];
    const size_t n = py_float_repr((double)value, buf);
    if (!out || out_bytes < n + 1) { set_error("c2v_format_float: buffer too small"); return C2V_EINVAL; }
    memcpy(out, buf, n); out[n] = 0;
    return (int)n;
}

int c2v_write_code_vectors(const char *vector_path, const char *mode, int64_t header_items, int64_t n, int32_t H,
                           const float *code_vectors, const int64_t *label, const char *names_blob,
                           const int64_t *name_offsets, int64_t n_names, const char *result_path, const char *result_mode,
                           const int64_t *ids, const int64_t *pred_label, const float *pred_score)
{
    if (!vector_path || !mode || n < 0 || H < 1 || (n && (!code_vectors || !label)) || !names_blob || !name_offsets) {
        set_error("c2v_write_code_vectors: bad argument");
        return C2V_EINVAL;
    }
    if (result_path && (!ids || !pred_label || !pred_score)) {
        set_error("c2v_write_code_vectors: the result file needs ids, pred_label and pred_score");
        return C2V_EINVAL;
    }
    for (int64_t i = 0; i < n; ++i) {
        if (label[i] < 0 || label[i] >= n_names || (result_path && (pred_label[i] < 0 || pred_label[i] >= n_names))) {
            set_error("c2v_write_code_vectors: row %lld: label index outside the vocabulary (KeyError in the reference)", (long long)i);
            return C2V_EINDEX;
        }
    }
    FILE *fv = fopen(vector_path, mode);
    if (!fv) { set_error("cannot open %s: %s", vector_path, strerror(errno)); return C2V_EINVAL; }
    FILE *fr = nullptr;
    if (result_path) {
        fr = fopen(result_path, result_mode ? result_mode : "w");
        if (!fr) { set_error("cannot open %s: %s", result_path, strerror(errno)); fclose(fv); return C2V_EINVAL; }
    }
    std::vector<char> vbuf(1 << 20), rbuf(1 << 16);
    setvbuf(fv, vbuf.data(), _IOFBF, vbuf.size());
    if (fr) setvbuf(fr, rbuf.data(), _IOFBF, rbuf.size());
    if (header_items >= 0) fprintf(fv, "%lld\t%d\n", (long long)header_items, (int)H);   // main.py:227-228
    std::string line;
    char num[48];
    bool ok = true;
    for (int64_t i = 0; i < n && ok; ++i) {
        const char *nm = names_blob + name_offsets[label[i]];
        const size_t nl = (size_t)(name_offsets[label[i] + 1] - name_offsets[label[i]]);
        line.assign(nm, nl);
        line.push_back('\t');
        const float *v = code_vectors + (size_t)i * H;
        for (int h = 0; h < H; ++h) {                           // main.py:416  " ".join(str(e.item()) for e in vec)
            if (h) line.push_back(' ');
            line.append(num, py_float_repr((double)v[h], num));
        }
        line.push_back('\n');
        ok = fwrite(line.data(), 1, line.size(), fv) == line.size();
        if (fr && ok) {                                          // main.py:420
            const char *pn = names_blob + name_offsets[pred_label[i]];
            const size_t pl = (size_t)(name_offsets[pred_label[i] + 1] - name_offsets[pred_label[i]]);
            const bool same = pl == nl && !memcmp(pn, nm, nl);
            line.assign(std::to_string((long long)ids[i]));
            line.push_back('\t');
            line.append(same ? "True" : "False");
            line.push_back('\t');
            line.append(nm, nl);
            line.push_back('\t');
            line.append(pn, pl);
            line.push_back('\t');
            line.append(num, py_float_repr((double)pred_score[i], num));
            line.push_back('\n');
            ok = fwrite(line.data(), 1, line.size(), fr) == line.size();
        }
    }
    if (fclose(fv) != 0) ok = false;
    if (fr && fclose(fr) != 0) ok = false;
    if (!ok) { set_error("short write to %s", vector_path); return C2V_EINVAL; }
    return C2V_OK;
}

}  // extern "C"

// ---- reading the vector file back (c2v_read_code_vectors) ------------------------------------------------------------
struct c2v_vectors {
    std::vector<float> vec;              // [n, H]
    std::vector<int64_t> name_off;       // [n + 1]
    std::string names;
    int64_t header_items = -1;
    int32_t H = 0;
};

namespace {

// `a\tb` with two integers (the header c2v_write_code_vectors writes)
bool is_header(const char *b, const char *e, long long *items, long long *H)
{
    const char *t = (const char *)memchr(b, '\t', (size_t)(e - b));
    return t && !memchr(t + 1, '\t', (size_t)(e - t - 1)) && parse_int(b, t, items) && parse_int(t + 1, e, H);
}

// one `name\tv0 v1 ...` line (without its '\n'); H < 0: the first data line, which sets H
bool read_vector_line(c2v_vectors *v, const char *b, const char *e, long long line_no, std::string *err)
{
    char msg[160];
    while (e > b && (e[-1] == '\r' || e[-1] == ' ')) --e;
    const char *t = (const char *)memchr(b, '\t', (size_t)(e - b));
    if (!t) {
        snprintf(msg, sizeof(msg), "line %lld: no tab between the name and the values", line_no);
        *err = msg;
        return false;
    }
    const size_t n0 = v->vec.size();
    const char *p = t + 1;
    while (true) {
        while (p < e && *p == ' ') ++p;
        if (p == e) break;
        double x = 0.0;
        // from_chars: correctly rounded like strtod, but independent of the process locale; it takes no leading '+'
        const auto r = std::from_chars(p + (*p == '+'), e, x);
        if (r.ec == std::errc::invalid_argument || (r.ptr < e && *r.ptr != ' ')) {
            snprintf(msg, sizeof(msg), "line %lld: value %zu is not a number", line_no, v->vec.size() - n0);
            *err = msg;
            return false;
        }
        if (r.ec == std::errc::result_out_of_range)      // what strtod returns there: +-HUGE_VAL or a denormal / zero
            x = strtod(std::string(p, r.ptr).c_str(), nullptr);
        v->vec.push_back((float)x);
        p = r.ptr;
    }
    const long long got = (long long)(v->vec.size() - n0);
    if (v->H == 0) v->H = (int32_t)got;
    if (got != v->H || got == 0) {
        snprintf(msg, sizeof(msg), "line %lld: %lld values, expected %d", line_no, got, v->H);
        *err = msg;
        return false;
    }
    v->names.append(b, (size_t)(t - b));
    v->name_off.push_back((int64_t)v->names.size());
    return true;
}

}  // namespace

extern "C" {

int c2v_read_code_vectors(const char *path, int32_t header, c2v_vectors **out)
{
    if (!path || !out || header < -1 || header > 1) { set_error("c2v_read_code_vectors: bad argument"); return C2V_EINVAL; }
    const int fd = open(path, O_RDONLY);
    if (fd < 0) { set_error("cannot open %s: %s", path, strerror(errno)); return C2V_EINVAL; }
    struct stat st;
    if (fstat(fd, &st) != 0) { set_error("fstat %s: %s", path, strerror(errno)); close(fd); return C2V_EINVAL; }
    const size_t size = (size_t)st.st_size;
    const char *m = nullptr;
    if (size > 0) {
        void *mp = mmap(nullptr, size, PROT_READ, MAP_PRIVATE, fd, 0);
        if (mp == MAP_FAILED) { set_error("mmap %s: %s", path, strerror(errno)); close(fd); return C2V_EINVAL; }
        madvise(mp, size, MADV_SEQUENTIAL);
        m = (const char *)mp;
    }
    close(fd);
    c2v_vectors *v = new c2v_vectors();
    v->name_off.push_back(0);
    std::string err;
    bool ok = true;
    long long line_no = 0;
    for (size_t pos = 0; pos < size && ok;) {
        const char *b = m + pos;
        const char *nl = (const char *)memchr(b, '\n', size - pos);
        const char *e = nl ? nl : m + size;
        pos = (size_t)(e - m) + 1;
        ++line_no;
        if (line_no == 1 && header != 0) {
            long long items = 0, H = 0;
            if (is_header(b, e, &items, &H)) {
                if (H < 1 || H > (1 << 20)) { err = "line 1: header encode_size out of range"; ok = false; break; }
                v->header_items = items; v->H = (int32_t)H;
                continue;
            }
            if (header == 1) { err = "line 1: expected the `n_items\\tencode_size` header"; ok = false; break; }
        }
        ok = read_vector_line(v, b, e, line_no, &err);
    }
    if (m) munmap((void *)m, size);
    if (!ok) { set_error("%s: %s", path, err.c_str()); delete v; return C2V_EINVAL; }
    *out = v;
    return C2V_OK;
}

int c2v_vectors_get_info(const c2v_vectors *v, c2v_vectors_info *info)
{
    if (!v || !info) { set_error("c2v_vectors_get_info: NULL argument"); return C2V_EINVAL; }
    info->n = (int64_t)(v->name_off.size() - 1);
    info->header_items = v->header_items;
    info->H = v->H; info->reserved = 0;
    info->name_bytes = (int64_t)v->names.size();
    return C2V_OK;
}

int c2v_vectors_export(const c2v_vectors *v, float *vectors, int64_t *name_offsets, char *name_blob)
{
    if (!v) { set_error("c2v_vectors_export: NULL handle"); return C2V_EINVAL; }
    if (vectors && !v->vec.empty()) memcpy(vectors, v->vec.data(), v->vec.size() * sizeof(float));
    if (name_offsets) memcpy(name_offsets, v->name_off.data(), v->name_off.size() * sizeof(int64_t));
    if (name_blob && !v->names.empty()) memcpy(name_blob, v->names.data(), v->names.size());
    return C2V_OK;
}

void c2v_vectors_free(c2v_vectors *v) { delete v; }

}  // extern "C"
