// Whole-model runtime of the C ABI: dh_model_inspect / load / input / forward / output / free (include/deephar_b200.h,
// "whole model").  The file is the launch list deephar_b200/export.py recorded from Model._bind_plan; this file parses
// it, checks every argument against the arenas it points into, relocates the (arena, offset) pointers onto one device
// allocation and replays the launches through the same entry points the Python host calls.
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include <string>
#include <vector>

#include "common.cuh"

namespace {

// entry-point ids of the file, and the tags of their arguments between ctx and stream (export.ENTRY_POINTS)
enum Entry {
    E_CONV, E_SEPCONV, E_MAXPOOL, E_UPSAMPLE_ADD, E_ADD_N, E_SAM2D, E_SAM2D_CTX, E_SAM3D, E_SAM3D_EX, E_KRON, E_ZEROPAD,
    E_MAXMIN_POOL, E_GLOBAL_MAXMIN_SOFTMAX, E_MASK_MUL, E_COUNT
};
const char* const kEntryName[E_COUNT] = {
    "dh_conv2d_f32", "dh_sepconv2d_f32", "dh_maxpool2d_f32", "dh_upsample2x_add_f32", "dh_add_n_f32",
    "dh_softargmax2d_f32", "dh_softargmax2d_ctx_f32", "dh_softargmax3d_f32", "dh_softargmax3d_ex_f32", "dh_kron_pool_f32",
    "dh_zeropad2d_f32", "dh_maxmin_pool2d_f32", "dh_global_maxmin_softmax_f32", "dh_mask_mul_f32"};
const char* const kEntrySig[E_COUNT] = {"vpwdv", "vppwdv", "viiiiiv", "vvv", "vippiv", "vvfippv", "viifpp",
                                         "viipp", "viifppv", "vvp", "viiv", "vv", "vp", "ppiip"};

const int kArenaWeights = 0, kArenaPacked = 1, kArenaWorkspace = 2, kArenaSlot0 = 3;
const int64_t kArenaAlign = 512;

// Until relocation a pointer holds its file reference: 0 = NULL, else (arena + 1) << 48 | byte offset.
const int kRefShift = 48;
const uint64_t kRefOffMask = (1ull << kRefShift) - 1;
typedef __int128 Wide;
inline int ref_arena(const void* p) { return (int)((uint64_t)(uintptr_t)p >> kRefShift) - 1; }

struct Arg {
    char tag;
    int64_t i;
    float f;
    uint64_t p;
    std::vector<dh_view> views;     // 'v'
    dh_conv_desc desc;              // 'd'
    dh_packed_w packed;             // 'w'
    int count;                      // 'v' / 'd' / 'w': structs recorded (0 = NULL pointer)
};

struct Launch {
    int entry;
    std::string label;
    std::vector<Arg> a;
};

struct Output {
    dh_view view;
    dh_model_output_info info;
};

const uint8_t kSlotFrame = 0, kSlotClip = 1;

struct Parsed {
    dh_model_info info;
    std::vector<uint8_t> weights, packed;
    std::vector<int64_t> arena_bytes;     // by arena id
    std::vector<uint8_t> slot_kind;       // by slot: kSlotFrame / kSlotClip (version 2; empty in version 1)
    dh_view input;
    std::vector<Output> outputs;
    std::vector<Launch> launches;
};

// A stream file (ClipStream.export).  Arenas: 0 weights, 1 packed, 2 / 3 the frame / clip stage's workspace, then the
// frame slots, the clip slots and the rings.
const int kArenaClipWorkspace = 3, kStreamSlot0 = 4;

struct StreamParsed {
    dh_stream_info info;
    std::vector<uint8_t> weights, packed;
    std::vector<int64_t> arena_bytes;
    int clip_slot0, ring0;                // first arena of the clip slots and of the rings
    std::vector<dh_clip_window> boundary;
    dh_view input;
    std::vector<Output> outputs;          // frame outputs, then clip outputs
    std::vector<Launch> frame, clip;
};

// Device memory after a stream's arenas (each 256-byte aligned): the window table, the clip-output views of
// dh_stream_ready_f32, the window kernel's counter pair, the per-stream counts and the ready flags.
struct StreamTail {
    int64_t table, outs, counter, counts, ready, end;
};
StreamTail stream_tail(int64_t base, int n_boundary, int n_clip_outputs, int S) {
    auto up = [](int64_t x) { return (x + 255) / 256 * 256; };
    StreamTail t;
    t.table = up(base);
    t.outs = up(t.table + (int64_t)n_boundary * sizeof(dh_clip_window));
    t.counter = up(t.outs + (int64_t)n_clip_outputs * sizeof(dh_view));
    t.counts = up(t.counter + 2 * sizeof(int32_t));
    t.ready = up(t.counts + (int64_t)S * sizeof(int32_t));
    t.end = up(t.ready + (int64_t)S * sizeof(int32_t));
    return t;
}

class Reader {
  public:
    Reader(const uint8_t* d, size_t n) : d_(d), n_(n), pos_(0) {}
    bool get(void* dst, size_t k) {
        if (k > n_ - pos_) return false;
        memcpy(dst, d_ + pos_, k);
        pos_ += k;
        return true;
    }
    template <typename T> bool get(T* v) { return get(v, sizeof(T)); }
    bool ptr(uint64_t* ref) {
        int32_t arena;
        int64_t off;
        if (!get(&arena) || !get(&off)) return false;
        if (arena == -1 && off == 0) { *ref = 0; return true; }
        if (arena < 0 || arena >= (1 << 14) || off < 0 || (uint64_t)off > kRefOffMask) { bad_ = true; return false; }
        *ref = ((uint64_t)(arena + 1) << kRefShift) | (uint64_t)off;
        return true;
    }
    bool view(dh_view* v) {
        uint64_t r;
        if (!ptr(&r) || !get(&v->n) || !get(&v->h) || !get(&v->w) || !get(&v->c) || !get(&v->ld)) return false;
        v->p = (float*)(uintptr_t)r;
        return true;
    }
    bool cptr(const float** p) {
        uint64_t r;
        if (!ptr(&r)) return false;
        *p = (const float*)(uintptr_t)r;
        return true;
    }
    bool desc(dh_conv_desc* d) {
        return get(&d->kh) && get(&d->kw) && get(&d->sh) && get(&d->sw) && get(&d->pad_same) && get(&d->pre_relu) &&
               get(&d->post_relu) && get(&d->n_res) && cptr(&d->pre_scale) && cptr(&d->pre_shift) &&
               cptr(&d->post_scale) && cptr(&d->post_shift) && view(&d->res[0]) && view(&d->res[1]) &&
               get(&d->precision) && get(&d->res_up2x) && view(&d->pool_out);
    }
    bool packed(dh_packed_w* w) {
        uint64_t hi, lo;
        if (!ptr(&hi) || !ptr(&lo) || !get(&w->cout_pad) || !get(&w->k)) return false;
        w->hi = (const void*)(uintptr_t)hi;
        w->lo = (const void*)(uintptr_t)lo;
        return true;
    }
    bool shape(int32_t* rank, int64_t* dims) {
        if (!get(rank)) return false;
        if (*rank < 1 || *rank > DH_MODEL_MAX_RANK) { bad_ = true; return false; }
        for (int i = 0; i < DH_MODEL_MAX_RANK; ++i) dims[i] = 0;
        for (int i = 0; i < *rank; ++i)
            if (!get(&dims[i])) return false;
        return true;
    }
    size_t left() const { return n_ - pos_; }
    bool bad() const { return bad_; }

  private:
    const uint8_t* d_;
    size_t n_, pos_;
    bool bad_ = false;
};

// The parser and the checks: < 0 with the error set, naming the launch.
class Checker {
  public:
    Checker(std::vector<int64_t>* arena_bytes, const char* file) : arenas_(arena_bytes), file_(file) {}

    // `bytes` from the pointer's offset must lie in its arena; float data must be 4-byte aligned.  Extents are products
    // of up to four 32-bit fields of the file: they are computed in 128 bits, where they cannot wrap.
    int ptr(uint64_t ref, Wide bytes, const char* what) {
        if (!ref) return 0;
        const int arena = (int)(ref >> kRefShift) - 1;
        const int64_t off = (int64_t)(ref & kRefOffMask);
        if (arena >= (int)arenas_->size()) return fail("%s points into arena %d of %d", what, arena,
                                                      (int)arenas_->size());
        if (!stage_arenas.empty() && !stage_arenas[arena])
            return fail("%s points into arena %d, outside the %s stage", what, arena, stage);
        if (off % 4) return fail("%s: byte offset %lld is not 4-byte aligned", what, (long long)off);
        const int64_t size = (*arenas_)[arena];
        if (bytes < 0 || off > size || bytes > (Wide)(size - off))
            return fail("%s: %.0f bytes at offset %lld overrun arena %d (%lld bytes)", what, (double)bytes,
                        (long long)off, arena, (long long)size);
        return 0;
    }
    int floats(const void* p, Wide count, const char* what) { return ptr((uint64_t)(uintptr_t)p, 4 * count, what); }
    int view(const dh_view& v, const char* what) {
        if (!v.p) return 0;
        if (v.n < 1 || v.h < 1 || v.w < 1 || v.c < 1 || v.ld < v.c)
            return fail("%s: bad view (n %d, h %d, w %d, c %d, ld %d)", what, v.n, v.h, v.w, v.c, v.ld);
        return floats(v.p, ((Wide)v.n * v.h * v.w - 1) * v.ld + v.c, what);
    }
    int range(int64_t v, int64_t lo, int64_t hi, const char* what) {
        if (v < lo || v > hi) return fail("%s = %lld is outside [%lld, %lld]", what, (long long)v, (long long)lo,
                                          (long long)hi);
        return 0;
    }
    int fail(const char* fmt, ...) __attribute__((format(printf, 2, 3)));

    int parse(const uint8_t* data, size_t n, Parsed* m);
    int parse_blobs(Reader& r, int use_tensor_cores, std::vector<uint8_t>* weights, std::vector<uint8_t>* packed);
    int parse_stream(const uint8_t* data, size_t n, StreamParsed* m);
    int parse_output(Reader& r, int k, Output* o, const char* what, const char* slots, int slot0, int slot_end,
                     int expect_n = -1);
    int parse_launches(Reader& r, const char* prefix, std::vector<Launch>* launches);
    int check_launch(const Launch& L);
    int check_items(const Parsed& m);

    const char* where = "header";
    std::string where_buf;
    // non-empty while a stream stage's launches are parsed: the arenas they may point into
    std::vector<char> stage_arenas;
    const char* stage = "";

  private:
    std::vector<int64_t>* arenas_;
    const char* file_;
};

int Checker::fail(const char* fmt, ...) {
    char msg[384];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(msg, sizeof(msg), fmt, ap);
    va_end(ap);
    dh_set_error("deephar_b200 %s file, %s: %s", file_, where, msg);
    return -1;
}

#define TRY(x)                       \
    do {                             \
        int rc__ = (x);              \
        if (rc__) return rc__;       \
    } while (0)
#define NEED(x)                                                                    \
    do {                                                                           \
        if (!(x)) return fail("%s", r.bad() ? "malformed field" : "truncated");    \
    } while (0)

// the weight and packed-operand arenas, as both formats store them
int Checker::parse_blobs(Reader& r, int use_tensor_cores, std::vector<uint8_t>* weights, std::vector<uint8_t>* packed) {
    int64_t wb, pb;
    NEED(r.get(&wb));
    if (wb < 0 || (uint64_t)wb > r.left()) return fail("truncated weight arena");
    weights->resize(wb);
    NEED(r.get(weights->data(), wb));
    NEED(r.get(&pb));
    if (pb < 0 || (uint64_t)pb > r.left()) return fail("truncated packed-operand arena");
    if (!use_tensor_cores && pb) return fail("packed operands in a file without tensor cores");
    packed->resize(pb);
    NEED(r.get(packed->data(), pb));
    return 0;
}

int Checker::parse(const uint8_t* data, size_t n, Parsed* m) {
    Reader r(data, n);
    dh_model_info& I = m->info;
    memset(&I, 0, sizeof(I));
    char magic[8];
    NEED(r.get(magic, 8));
    if (memcmp(magic, "DHMODEL\0", 8)) return fail("not a deephar_b200 model file (bad magic)");
    uint32_t version;
    NEED(r.get(&version));
    if (version < 1 || version > DH_MODEL_VERSION)
        return fail("format version %u; this library reads versions 1 to %d", version, DH_MODEL_VERSION);
    I.version = (int32_t)version;
    NEED(r.get(&I.precision) && r.get(&I.use_tensor_cores) && r.get(&I.frame_items) && r.get(&I.clip_items) &&
         r.get(&I.frames_per_clip));
    TRY(range(I.precision, 0, 3, "precision"));
    TRY(range(I.use_tensor_cores, 0, 1, "use_tensor_cores"));
    TRY(range(I.frames_per_clip, 1, 1 << 20, "frames_per_clip"));
    TRY(range(I.frame_items, 1, 1 << 30, "frame_items"));
    TRY(range(I.clip_items, 0, I.frame_items, "clip_items"));
    NEED(r.shape(&I.input_rank, I.input_shape));
    TRY(parse_blobs(r, I.use_tensor_cores, &m->weights, &m->packed));
    const int64_t wb = m->weights.size(), pb = m->packed.size();
    int32_t slots;
    NEED(r.get(&slots));
    if (slots < 1 || (uint64_t)slots * 8 > r.left()) return fail(slots < 1 ? "no activation slot" : "truncated");
    m->arena_bytes.assign(kArenaSlot0 + slots, 0);
    m->arena_bytes[kArenaWeights] = wb;
    m->arena_bytes[kArenaPacked] = pb;
    I.weight_bytes = wb;
    I.packed_bytes = pb;
    I.n_slots = slots;
    const int64_t kMaxArena = 1ll << 40;
    for (int s = 0; s < slots; ++s) {
        int64_t b;
        NEED(r.get(&b));
        if (b < 0 || b > kMaxArena || b % 4) return fail("slot %d: bad size %lld", s, (long long)b);
        m->arena_bytes[kArenaSlot0 + s] = b;
        I.activation_bytes += b;
    }
    if (version >= 2) {
        m->slot_kind.resize(slots);
        NEED(r.get(m->slot_kind.data(), slots));
        for (int s = 0; s < slots; ++s)
            if (m->slot_kind[s] != kSlotFrame && m->slot_kind[s] != kSlotClip)
                return fail("slot %d: kind %u (0 = frame, 1 = clip)", s, m->slot_kind[s]);
    }
    NEED(r.get(&I.workspace_bytes));
    if (I.workspace_bytes < 0 || I.workspace_bytes > kMaxArena) return fail("bad workspace size");
    m->arena_bytes[kArenaWorkspace] = I.workspace_bytes;
    for (int a = 0; a < (int)m->arena_bytes.size(); ++a)
        I.device_bytes += (m->arena_bytes[a] + kArenaAlign - 1) / kArenaAlign * kArenaAlign;

    where = "input";
    NEED(r.view(&m->input));
    TRY(view(m->input, "input view"));
    if (!m->input.p || m->input.ld != m->input.c || ref_arena(m->input.p) < kArenaSlot0)
        return fail("the input must be a dense view of an activation slot");
    where = "outputs";
    int32_t nout;
    NEED(r.get(&nout));
    if (nout < 1 || nout > (1 << 16)) return fail("%d outputs", nout);
    I.n_outputs = nout;
    m->outputs.resize(nout);
    for (int k = 0; k < nout; ++k)
        TRY(parse_output(r, k, &m->outputs[k], "output", "an activation slot", kArenaSlot0, (int)m->arena_bytes.size()));
    TRY(parse_launches(r, "", &m->launches));
    I.n_launches = (int64_t)m->launches.size();
    where = "end";
    if (r.left()) return fail("%zu bytes after the last launch", r.left());
    return version >= 2 ? check_items(*m) : 0;
}

// One output record: its view must lie in arenas [slot0, slot_end) (`slots` names them) and have expect_n items (if
// >= 0); its shape must hold the view.
int Checker::parse_output(Reader& r, int k, Output* out, const char* what, const char* slots, int slot0, int slot_end,
                          int expect_n) {
    Output& o = *out;
    memset(&o.info, 0, sizeof(o.info));
    NEED(r.view(&o.view));
    TRY(view(o.view, "output view"));
    if (!o.view.p || ref_arena(o.view.p) < slot0 || ref_arena(o.view.p) >= slot_end)
        return fail("%s %d is not a view of %s", what, k, slots);
    if (expect_n >= 0 && o.view.n != expect_n) return fail("%s %d has n = %d, expected S = %d", what, k, o.view.n, expect_n);
    NEED(r.shape(&o.info.rank, o.info.shape));
    int64_t elems = 1;
    for (int i = 0; i < o.info.rank; ++i) {
        if (o.info.shape[i] < 1 || o.info.shape[i] > (1ll << 31)) return fail("%s %d: bad shape", what, k);
        elems *= o.info.shape[i];
        if (elems > (1ll << 40)) return fail("%s %d: bad shape", what, k);
    }
    if ((__int128)elems != (__int128)o.view.n * o.view.h * o.view.w * o.view.c)
        return fail("%s %d: shape does not hold its view", what, k);
    int32_t len;
    NEED(r.get(&len));
    if (len < 0 || (uint64_t)len > r.left()) return fail("truncated output name");
    std::string name(len, '\0');
    NEED(r.get(&name[0], len));
    snprintf(o.info.name, sizeof(o.info.name), "%s", name.c_str());
    return 0;
}

// i32 L, then L launch records, each checked (check_launch).  prefix names the list in messages: "" or "frame ".
int Checker::parse_launches(Reader& r, const char* prefix, std::vector<Launch>* launches) {
    where_buf = std::string(prefix) + "launches";
    where = where_buf.c_str();
    int32_t nl;
    NEED(r.get(&nl));
    if (nl < 1 || nl > (1 << 20)) return fail("%d launches", nl);
    launches->resize(nl);
    for (int i = 0; i < nl; ++i) {
        Launch& L = (*launches)[i];
        int32_t nargs, len;
        where_buf = std::string(prefix) + "launch " + std::to_string(i);
        where = where_buf.c_str();
        NEED(r.get(&L.entry) && r.get(&nargs) && r.get(&len));
        if (L.entry < 0 || L.entry >= E_COUNT) return fail("unknown entry point %d", L.entry);
        if (len < 0 || (uint64_t)len > r.left()) return fail("truncated label");
        L.label.assign(len, '\0');
        NEED(r.get(&L.label[0], len));
        where_buf = std::string(prefix) + "launch " + std::to_string(i) + " (" + L.label + ")";
        where = where_buf.c_str();
        const char* sig = kEntrySig[L.entry];
        if (nargs != (int)strlen(sig)) return fail("%d arguments; %s takes %d", nargs, kEntryName[L.entry],
                                                   (int)strlen(sig));
        L.a.resize(nargs);
        for (int k = 0; k < nargs; ++k) {
            Arg& a = L.a[k];
            uint8_t tag;
            NEED(r.get(&tag));
            if (tag != (uint8_t)sig[k]) return fail("argument %d has tag '%c'; %s expects '%c'", k, tag,
                                                    kEntryName[L.entry], sig[k]);
            a.tag = (char)tag;
            a.count = 0;
            if (tag == 'i') NEED(r.get(&a.i));
            else if (tag == 'f') NEED(r.get(&a.f));
            else if (tag == 'p') NEED(r.ptr(&a.p));
            else {
                NEED(r.get(&a.count));
                const int maxc = tag == 'v' ? 4 : 1;
                if (a.count < 0 || a.count > maxc) return fail("argument %d: %d structs", k, a.count);
                for (int j = 0; j < a.count; ++j) {
                    if (tag == 'v') {
                        dh_view v;
                        NEED(r.view(&v));
                        a.views.push_back(v);
                    } else if (tag == 'd') {
                        NEED(r.desc(&a.desc));
                    } else {
                        NEED(r.packed(&a.packed));
                    }
                }
            }
        }
        TRY(check_launch(L));
    }
    return 0;
}

int Checker::parse_stream(const uint8_t* data, size_t n, StreamParsed* m) {
    Reader r(data, n);
    dh_stream_info& I = m->info;
    memset(&I, 0, sizeof(I));
    char magic[9];
    NEED(r.get(magic, 9));
    if (memcmp(magic, "DHSTREAM\0", 9)) return fail("not a deephar_b200 stream file (bad magic)");
    uint32_t version;
    NEED(r.get(&version));
    if (version != DH_STREAM_VERSION)
        return fail("format version %u; this library reads version %d", version, DH_STREAM_VERSION);
    I.version = (int32_t)version;
    NEED(r.get(&I.precision) && r.get(&I.use_tensor_cores) && r.get(&I.n_streams) && r.get(&I.frames_per_clip));
    TRY(range(I.precision, 0, 3, "precision"));
    TRY(range(I.use_tensor_cores, 0, 1, "use_tensor_cores"));
    TRY(range(I.n_streams, 1, 1 << 20, "S"));
    TRY(range(I.frames_per_clip, 2, 1 << 20, "T"));
    const int S = I.n_streams, T = I.frames_per_clip;
    TRY(range((int64_t)S * T, 1, 1 << 30, "S*T"));
    NEED(r.shape(&I.input_rank, I.input_shape));
    if (I.input_rank != 4 || I.input_shape[0] != S || I.input_shape[3] != 3) return fail("input shape is not (S, H, W, 3)");
    TRY(parse_blobs(r, I.use_tensor_cores, &m->weights, &m->packed));
    I.weight_bytes = m->weights.size();
    I.packed_bytes = m->packed.size();
    m->arena_bytes.assign(kStreamSlot0, 0);
    m->arena_bytes[kArenaWeights] = I.weight_bytes;
    m->arena_bytes[kArenaPacked] = I.packed_bytes;
    const int64_t kMaxArena = 1ll << 40;
    // i32 count + i64 sizes of one group of arenas (a stage's slots, or the rings), appended to arena_bytes
    auto sizes = [&](const char* what, int64_t* count, int64_t* total) -> int {
        int32_t k;
        NEED(r.get(&k));
        if (k < 1 || k > (1 << 16)) return fail("%d %ss", k, what);
        if ((uint64_t)k * 8 > r.left()) return fail("truncated");
        *count = k;
        for (int s = 0; s < k; ++s) {
            int64_t b;
            NEED(r.get(&b));
            if (b < 0 || b > kMaxArena || b % 4) return fail("%s %d: bad size %lld", what, s, (long long)b);
            m->arena_bytes.push_back(b);
            *total += b;
        }
        return 0;
    };
    auto workspace = [&](int arena, int64_t* bytes) -> int {
        NEED(r.get(bytes));
        if (*bytes < 0 || *bytes > kMaxArena) return fail("bad workspace size");
        m->arena_bytes[arena] = *bytes;
        return 0;
    };
    where = "frame stage";
    TRY(sizes("frame slot", &I.n_frame_slots, &I.activation_bytes));
    TRY(workspace(kArenaWorkspace, &I.frame_workspace_bytes));
    m->clip_slot0 = (int)m->arena_bytes.size();
    where = "clip stage";
    TRY(sizes("clip slot", &I.n_clip_slots, &I.activation_bytes));
    TRY(workspace(kArenaClipWorkspace, &I.clip_workspace_bytes));
    m->ring0 = (int)m->arena_bytes.size();
    where = "rings";
    int64_t nb = 0;
    TRY(sizes("ring", &nb, &I.ring_bytes));
    I.n_boundary = (int32_t)nb;
    const int frame0 = kStreamSlot0, clip0 = m->clip_slot0, ring0 = m->ring0, end = (int)m->arena_bytes.size();
    auto in = [](const void* p, int lo, int hi) { return p && ref_arena(p) >= lo && ref_arena(p) < hi; };

    m->boundary.resize(nb);
    for (int b = 0; b < nb; ++b) {
        where_buf = "boundary " + std::to_string(b);
        where = where_buf.c_str();
        dh_clip_window& e = m->boundary[b];
        uint64_t ring;
        NEED(r.view(&e.src) && r.view(&e.dst) && r.ptr(&ring));
        e.ring = (float*)(uintptr_t)ring;
        TRY(view(e.src, "src"));
        TRY(view(e.dst, "dst"));
        if (!in(e.src.p, frame0, clip0)) return fail("src is not a view of a frame-stage slot");
        if (!in(e.dst.p, clip0, ring0)) return fail("dst is not a view of a clip-stage slot");
        if (e.src.n != S) return fail("src has n = %d, expected S = %d", e.src.n, S);
        if ((int64_t)e.dst.n != (int64_t)S * T) return fail("dst has n = %d, expected S*T = %lld", e.dst.n, (long long)S * T);
        if (e.src.h != e.dst.h || e.src.w != e.dst.w || e.src.c != e.dst.c)
            return fail("src (h %d, w %d, c %d) and dst (h %d, w %d, c %d) differ", e.src.h, e.src.w, e.src.c, e.dst.h,
                        e.dst.w, e.dst.c);
        if (!in(e.ring, ring0, end) || (ring & kRefOffMask)) return fail("the ring is not the start of a ring arena");
        const Wide want = (Wide)4 * S * T * e.src.h * e.src.w * e.src.c;
        if ((Wide)m->arena_bytes[ref_arena(e.ring)] != want)
            return fail("ring arena %d holds %lld bytes; S*T*h*w*c floats are %.0f bytes", ref_arena(e.ring),
                        (long long)m->arena_bytes[ref_arena(e.ring)], (double)want);
    }
    // The window kernel writes dst and ring and reads src: no write may touch what another entry reads or writes.
    // Views of one buffer with the same ld and disjoint channel windows (a concatenation) do not overlap.
    struct Span { int arena; int64_t off, bytes, ld, c; bool written; const char* what; int b; };
    std::vector<Span> spans;
    auto span = [](const dh_view& v, bool written, const char* what, int b) {
        const uint64_t ref = (uint64_t)(uintptr_t)v.p;
        return Span{ref_arena(v.p), (int64_t)(ref & kRefOffMask), 4 * (((int64_t)v.n * v.h * v.w - 1) * v.ld + v.c),
                    v.ld, v.c, written, what, b};
    };
    for (int b = 0; b < nb; ++b) {
        const dh_clip_window& e = m->boundary[b];
        spans.push_back(span(e.src, false, "src", b));
        spans.push_back(span(e.dst, true, "dst", b));
        spans.push_back(Span{ref_arena(e.ring), 0, m->arena_bytes[ref_arena(e.ring)], 1, 1, true, "ring", b});
    }
    where = "boundary table";
    for (size_t i = 0; i < spans.size(); ++i)
        for (size_t j = i + 1; j < spans.size(); ++j) {
            const Span &x = spans[i], &y = spans[j];
            if (!(x.written || y.written) || x.arena != y.arena) continue;
            if (x.off + x.bytes <= y.off || y.off + y.bytes <= x.off) continue;
            if (x.ld == y.ld && x.ld > 1) {
                const int64_t cx = x.off / 4 % x.ld, cy = y.off / 4 % y.ld;
                if (cx + x.c <= x.ld && cy + y.c <= y.ld && (cx + x.c <= cy || cy + y.c <= cx)) continue;
            }
            return fail("boundary %d %s and boundary %d %s overlap", x.b, x.what, y.b, y.what);
        }

    where = "input";
    NEED(r.view(&m->input));
    TRY(view(m->input, "input view"));
    if (!in(m->input.p, frame0, clip0) || m->input.ld != m->input.c || m->input.n != S ||
        m->input.h != I.input_shape[1] || m->input.w != I.input_shape[2] || m->input.c != 3)
        return fail("the input must be a dense (S, H, W, 3) view of a frame-stage slot");
    for (int clip = 0; clip < 2; ++clip) {
        where = clip ? "clip outputs" : "frame outputs";
        int32_t nout;
        NEED(r.get(&nout));
        if (nout < clip || nout > (1 << 16)) return fail("%d outputs", nout);
        (clip ? I.n_clip_outputs : I.n_frame_outputs) = nout;
        const char* what = clip ? "clip output" : "frame output";
        for (int k = 0; k < nout; ++k) {
            Output o;
            TRY(clip ? parse_output(r, k, &o, what, "a clip-stage slot", clip0, ring0, S)
                     : parse_output(r, k, &o, what, "a frame-stage slot", frame0, clip0, S));
            if (o.info.rank < 2 || o.info.shape[0] != S) return fail("%s %d: shape is not (S, ...)", what, k);
            m->outputs.push_back(o);
        }
    }
    for (int clip = 0; clip < 2; ++clip) {
        stage_arenas.assign(end, 0);
        stage_arenas[kArenaWeights] = stage_arenas[kArenaPacked] = 1;
        stage_arenas[clip ? kArenaClipWorkspace : kArenaWorkspace] = 1;
        for (int a = clip ? clip0 : frame0; a < (clip ? ring0 : clip0); ++a) stage_arenas[a] = 1;
        stage = clip ? "clip" : "frame";
        TRY(parse_launches(r, clip ? "clip " : "frame ", clip ? &m->clip : &m->frame));
    }
    stage_arenas.clear();
    I.n_frame_launches = (int64_t)m->frame.size();
    I.n_clip_launches = (int64_t)m->clip.size();
    where = "end";
    if (r.left()) return fail("%zu bytes after the last launch", r.left());
    int64_t base = 0;
    for (int64_t b : m->arena_bytes) base += (b + kArenaAlign - 1) / kArenaAlign * kArenaAlign;
    I.device_bytes = stream_tail(base, (int)nb, I.n_clip_outputs, S).end;
    return 0;
}

// Integer ranges, struct counts and the extent of every pointer an entry point reads or writes.
int Checker::check_launch(const Launch& L) {
    const std::vector<Arg>& a = L.a;
    const char* sig = kEntrySig[L.entry];
    for (size_t k = 0; k < a.size(); ++k) {
        if (sig[k] == 'v')
            for (const dh_view& v : a[k].views) TRY(view(v, "view"));
        if (sig[k] == 'i' && L.entry != E_MASK_MUL) TRY(range(a[k].i, -(1ll << 31), (1ll << 31) - 1, "integer"));
    }
    auto one = [&](int k, const char* what) -> int {
        if (a[k].count != 1 || !a[k].views[0].p) return fail("%s: one non-NULL view expected", what);
        return 0;
    };
    auto opt = [&](int k, const char* what) -> int {      // a view pointer that may be NULL
        if (a[k].count > 1) return fail("%s: at most one view", what);
        return 0;
    };
    auto vw = [&](int k) -> const dh_view& { return a[k].views[0]; };
    switch (L.entry) {
    case E_CONV:
    case E_SEPCONV: {
        const bool sep = L.entry == E_SEPCONV;
        const int kd = sep ? 4 : 3, kw = sep ? 3 : 2, ko = sep ? 5 : 4;
        TRY(one(0, "x"));
        TRY(one(ko, "out"));
        if (a[kd].count != 1) return fail("no conv descriptor");
        const dh_conv_desc& d = a[kd].desc;
        TRY(range(d.kh, 1, 31, "kh"));
        TRY(range(d.kw, 1, 31, "kw"));
        TRY(range(d.sh, 1, 8, "sh"));
        TRY(range(d.sw, 1, 8, "sw"));
        TRY(range(d.pad_same, 0, 1, "pad_same"));
        TRY(range(d.pre_relu, 0, 1, "pre_relu"));
        TRY(range(d.post_relu, 0, 1, "post_relu"));
        TRY(range(d.n_res, 0, 2, "n_res"));
        TRY(range(d.res_up2x, 0, 3, "res_up2x"));
        if (d.precision != 0 && d.precision != 1 && d.precision != 3) return fail("precision %d", d.precision);
        const Wide cin = vw(0).c, cout = vw(ko).c, taps = (Wide)d.kh * d.kw;
        if (sep) {
            if (!a[1].p || !a[2].p) return fail("NULL weights");
            TRY(floats((void*)(uintptr_t)a[1].p, taps * cin, "depthwise weights"));
            TRY(floats((void*)(uintptr_t)a[2].p, cin * cout, "pointwise weights"));
        } else {
            if (!a[1].p) return fail("NULL weights");
            TRY(floats((void*)(uintptr_t)a[1].p, taps * cin * cout, "weights"));
        }
        TRY(floats(d.pre_scale, cin, "pre_scale"));
        TRY(floats(d.pre_shift, cin, "pre_shift"));
        TRY(floats(d.post_scale, cout, "post_scale"));
        TRY(floats(d.post_shift, cout, "post_shift"));
        for (int i = 0; i < 2; ++i) TRY(view(d.res[i], "residual"));
        TRY(view(d.pool_out, "pool_out"));
        if (a[kw].count) {
            const dh_packed_w& w = a[kw].packed;
            if (w.cout_pad < 1 || w.k < 1 || w.cout_pad > (1 << 20) || w.k > (1 << 24)) return fail("packed geometry");
            TRY(ptr((uint64_t)(uintptr_t)w.hi, (Wide)2 * w.cout_pad * w.k, "packed hi"));
            TRY(ptr((uint64_t)(uintptr_t)w.lo, (Wide)2 * w.cout_pad * w.k, "packed lo"));
        }
        return 0;
    }
    case E_MAXPOOL:
        TRY(one(0, "x"));
        TRY(one(6, "out"));
        for (int k = 1; k <= 4; ++k) TRY(range(a[k].i, 1, 16, "pool size / stride"));
        return range(a[5].i, 0, 1, "pad_same");
    case E_UPSAMPLE_ADD:
        TRY(opt(0, "a"));
        TRY(one(1, "b"));
        return one(2, "out");
    case E_ADD_N: {
        TRY(range(a[1].i, 1, 4, "n_in"));
        if (a[0].count != a[1].i) return fail("%d views for n_in = %lld", a[0].count, (long long)a[1].i);
        TRY(one(5, "out"));
        if (!a[2].p != !a[3].p) return fail("scale and shift must come together");
        TRY(ptr(a[2].p, (Wide)4 * vw(5).c, "scale"));
        TRY(ptr(a[3].p, (Wide)4 * vw(5).c, "shift"));
        return range(a[4].i, 0, 1, "relu");
    }
    case E_SAM2D: {
        TRY(one(0, "h"));
        TRY(opt(1, "d"));
        TRY(opt(6, "prob_out"));
        TRY(range(a[3].i, 0, 1, "conf_on_prob"));
        const Wide nc = (Wide)vw(0).n * vw(0).c;
        const bool z = a[1].count && vw(1).p;
        if (!a[4].p || !a[5].p) return fail("NULL output");
        TRY(ptr(a[4].p, 4 * nc * (z ? 3 : 2), "out_pose"));
        return ptr(a[5].p, 4 * nc, "out_conf");
    }
    case E_SAM2D_CTX: {
        TRY(one(0, "h"));
        TRY(range(a[1].i, 1, 4096, "nj"));
        TRY(range(a[2].i, 0, 4096, "n_ctx"));
        const Wide nj = (Wide)vw(0).n * a[1].i;
        if (!a[4].p || !a[5].p) return fail("NULL output");
        TRY(ptr(a[4].p, 4 * nj * 2, "out_pose"));
        return ptr(a[5].p, 4 * nj, "out_vis");
    }
    case E_SAM3D:
    case E_SAM3D_EX: {
        TRY(one(0, "h"));
        TRY(range(a[1].i, 1, 4096, "nj"));
        TRY(range(a[2].i, 1, 4096, "depth_maps"));
        const int ko = L.entry == E_SAM3D ? 3 : 4;
        if (L.entry == E_SAM3D_EX) TRY(opt(6, "prob_out"));
        const Wide nj = (Wide)vw(0).n * a[1].i;
        if (!a[ko].p || !a[ko + 1].p) return fail("NULL output");
        TRY(ptr(a[ko].p, 4 * nj * 3, "out_pose"));
        return ptr(a[ko + 1].p, 4 * nj, "out_vis");
    }
    case E_KRON:
        TRY(one(0, "p"));
        TRY(one(1, "z"));
        if (!a[2].p) return fail("NULL output");
        return ptr(a[2].p, (Wide)4 * vw(0).n * vw(0).c * vw(1).c, "out");
    case E_ZEROPAD:
        TRY(one(0, "x"));
        TRY(one(3, "out"));
        TRY(range(a[1].i, 0, 1 << 16, "top"));
        return range(a[2].i, 0, 1 << 16, "left");
    case E_MAXMIN_POOL:
        TRY(one(0, "x"));
        return one(1, "out");
    case E_GLOBAL_MAXMIN_SOFTMAX:
        TRY(one(0, "x"));
        if (!a[1].p) return fail("NULL output");
        return ptr(a[1].p, (Wide)4 * vw(0).n * vw(0).c, "out");
    case E_MASK_MUL: {
        TRY(range(a[2].i, 1, 1ll << 36, "rows"));
        TRY(range(a[3].i, 1, 1 << 16, "dim"));
        if (!a[0].p || !a[1].p || !a[4].p) return fail("NULL argument");
        TRY(ptr(a[0].p, (Wide)4 * a[2].i * a[3].i, "p"));
        TRY(ptr(a[1].p, (Wide)4 * a[2].i, "c"));
        return ptr(a[4].p, (Wide)4 * a[2].i * a[3].i, "out");
    }
    }
    return fail("unknown entry point");
}

// Version 2, what dh_model_set_batch relies on: T * clip_items = frame_items; every view into an activation slot holds
// the exported item count of its slot's kind -- N clips in a clip slot, N * T frames in a frame slot, or N clips of T
// frames where frames_to_clip reads a frame slot as clips -- and dh_mask_mul_f32's rows over a slot are a multiple of N.
// So each scales by n / N.
int Checker::check_items(const Parsed& m) {
    const dh_model_info& I = m.info;
    const int64_t N = I.clip_items, T = I.frames_per_clip;
    if (N * T != I.frame_items)
        return fail("frame_items %d is not clip_items %d x frames_per_clip %d", I.frame_items, I.clip_items,
                    I.frames_per_clip);
    auto items = [&](const dh_view& v, const char* what) -> int {
        const int a = ref_arena(v.p);
        if (!v.p || a < kArenaSlot0) return 0;
        const int s = a - kArenaSlot0;
        const bool clip = m.slot_kind[s] == kSlotClip;
        if (v.n == N || (!clip && v.n == N * T)) return 0;
        return clip ? fail("%s has n = %d in clip slot %d, which holds %lld clips", what, v.n, s, (long long)N)
                    : fail("%s has n = %d in frame slot %d, which holds %lld frames (%lld clips)", what, v.n, s,
                           (long long)(N * T), (long long)N);
    };
    where = "input";
    TRY(items(m.input, "the input view"));
    where = "outputs";
    for (size_t k = 0; k < m.outputs.size(); ++k) {
        const Output& o = m.outputs[k];
        where_buf = "output " + std::to_string(k) + " (" + o.info.name + ")";
        where = where_buf.c_str();
        TRY(items(o.view, "its view"));
        if (o.info.shape[0] != N) return fail("shape[0] = %lld; the file's batch is %lld", (long long)o.info.shape[0],
                                              (long long)N);
    }
    for (size_t i = 0; i < m.launches.size(); ++i) {
        const Launch& L = m.launches[i];
        where_buf = "launch " + std::to_string(i) + " (" + L.label + ")";
        where = where_buf.c_str();
        for (size_t k = 0; k < L.a.size(); ++k) {
            const Arg& a = L.a[k];
            for (const dh_view& v : a.views) TRY(items(v, ("the view of argument " + std::to_string(k)).c_str()));
            if (a.tag == 'd' && a.count) {
                TRY(items(a.desc.res[0], "residual 0"));
                TRY(items(a.desc.res[1], "residual 1"));
                TRY(items(a.desc.pool_out, "pool_out"));
            }
        }
        if (L.entry == E_MASK_MUL && ref_arena((void*)(uintptr_t)L.a[0].p) >= kArenaSlot0 && L.a[2].i % N)
            return fail("rows = %lld is not a multiple of the batch %lld", (long long)L.a[2].i, (long long)N);
    }
    return 0;
}

int read_file(const char* path, const char* file, std::vector<uint8_t>* buf) {
    DH_CHECK_ARG(path != nullptr, "deephar_b200 %s file: path is NULL", file);
    FILE* f = fopen(path, "rb");
    DH_CHECK_ARG(f != nullptr, "deephar_b200 %s file %s: cannot open", file, path);
    uint8_t chunk[1 << 16];
    size_t n;
    while ((n = fread(chunk, 1, sizeof(chunk), f)) > 0) buf->insert(buf->end(), chunk, chunk + n);
    const bool err = ferror(f);
    fclose(f);
    DH_CHECK_ARG(!err, "deephar_b200 %s file %s: read error", file, path);
    return 0;
}

int parse_file(const char* path, Parsed* m) {
    std::vector<uint8_t> data;
    TRY(read_file(path, "model", &data));
    Checker ck(&m->arena_bytes, "model");
    return ck.parse(data.data(), data.size(), m);
}

int parse_stream_file(const char* path, StreamParsed* m) {
    std::vector<uint8_t> data;
    TRY(read_file(path, "stream", &data));
    Checker ck(&m->arena_bytes, "stream");
    return ck.parse_stream(data.data(), data.size(), m);
}

// ---- relocation ----------------------------------------------------------------------------------------------------------
struct Relocator {
    std::vector<uint8_t*> base;     // by arena id
    template <typename T> void fix(T*& p) const {
        const uint64_t ref = (uint64_t)(uintptr_t)p;
        p = ref ? (T*)(base[(ref >> kRefShift) - 1] + (ref & kRefOffMask)) : nullptr;
    }
    void fix(dh_view& v) const { fix(v.p); }
};

// One allocation of `total` bytes on ctx's device: the arenas (kArenaAlign-aligned) from its start, the weights and
// packed operands uploaded, everything from arena 2 (the first workspace) to the end zeroed.  Errors are reported as
// "<fn>: <cuda error>" and free what was allocated.
int upload(dh_ctx* ctx, const char* fn, int64_t total, const std::vector<int64_t>& arena_bytes,
           const std::vector<uint8_t>& weights, const std::vector<uint8_t>& packed, void** dev, Relocator* R) {
    *dev = nullptr;
    int prev = 0;
    cudaGetDevice(&prev);
    cudaError_t e = cudaSetDevice(ctx->device);
    if (e == cudaSuccess) e = cudaMalloc(dev, (size_t)total);
    if (e == cudaSuccess) {
        uint8_t* p = (uint8_t*)*dev;
        for (int64_t b : arena_bytes) {
            R->base.push_back(p);
            p += (b + kArenaAlign - 1) / kArenaAlign * kArenaAlign;
        }
        if (!weights.empty()) e = cudaMemcpy(R->base[kArenaWeights], weights.data(), weights.size(), cudaMemcpyHostToDevice);
        if (e == cudaSuccess && !packed.empty())
            e = cudaMemcpy(R->base[kArenaPacked], packed.data(), packed.size(), cudaMemcpyHostToDevice);
        if (e == cudaSuccess)      // activations start zeroed, so a forward's result never depends on earlier memory
            e = cudaMemset(R->base[kArenaWorkspace], 0, (size_t)(total - (R->base[kArenaWorkspace] - (uint8_t*)*dev)));
        if (e == cudaSuccess) e = cudaDeviceSynchronize();
    }
    cudaSetDevice(prev);
    if (e != cudaSuccess) {
        dh_set_error("%s: %s", fn, cudaGetErrorString(e));
        if (*dev) cudaFree(*dev);
        *dev = nullptr;
        return (int)e;
    }
    return 0;
}

// Relocate every pointer of a launch list and plan each convolution as the library would run it, within `workspace`
// bytes.  what: how messages name the list's launches ("dh_model_load: launch").
int relocate_and_plan(dh_ctx* ctx, const Relocator& R, std::vector<Launch>* launches, int64_t workspace,
                      const char* what) {
    int rc = 0;
    for (size_t i = 0; i < launches->size() && !rc; ++i) {
        Launch& L = (*launches)[i];
        for (Arg& a : L.a) {
            if (a.tag == 'p') {
                float* p = (float*)(uintptr_t)a.p;
                R.fix(p);
                a.p = (uint64_t)(uintptr_t)p;
            }
            for (dh_view& v : a.views) R.fix(v);
            if (a.tag == 'd' && a.count) {
                R.fix(a.desc.pre_scale);
                R.fix(a.desc.pre_shift);
                R.fix(a.desc.post_scale);
                R.fix(a.desc.post_shift);
                R.fix(a.desc.res[0]);
                R.fix(a.desc.res[1]);
                R.fix(a.desc.pool_out);
            }
            if (a.tag == 'w' && a.count) {
                R.fix(a.packed.hi);
                R.fix(a.packed.lo);
            }
        }
        if (L.entry == E_CONV || L.entry == E_SEPCONV) {
            // the library's choice for this layer, as Model._bind asks for it: a layer no kernel takes fails here
            const bool sep = L.entry == E_SEPCONV;
            const std::vector<Arg>& a = L.a;
            const int kw = sep ? 3 : 2;
            const dh_packed_w* pw = a[kw].count ? &a[kw].packed : nullptr;
            dh_conv_plan_info info;
            rc = sep ? dh_sepconv2d_plan(ctx, &a[0].views[0], (const float*)(uintptr_t)a[1].p,
                                         (const float*)(uintptr_t)a[2].p, pw, &a[4].desc, &a[5].views[0], &info)
                     : dh_conv2d_plan(ctx, &a[0].views[0], (const float*)(uintptr_t)a[1].p, pw, &a[3].desc,
                                      &a[4].views[0], &info);
            char msg[512];
            if (rc) {
                snprintf(msg, sizeof(msg), "%s", dh_last_error());
                dh_set_error("%s %zu (%s): no kernel takes it: %s", what, i, L.label.c_str(), msg);
            } else if (info.workspace_bytes > workspace) {
                dh_set_error("%s %zu (%s) needs %lld workspace bytes, the file has %lld", what, i, L.label.c_str(),
                             (long long)info.workspace_bytes, (long long)workspace);
                rc = -1;
            }
        }
    }
    return rc < 0 ? rc : (rc ? -1 : 0);
}

// Set ctx's workspace and issue a launch list on `stream`.  what: how messages name its launches.
int issue(dh_ctx* ctx, const std::vector<Launch>& launches, void* workspace, int64_t workspace_bytes, void* stream,
          const char* what) {
    TRY(dh_set_workspace(ctx, workspace, workspace_bytes));
    for (size_t i = 0; i < launches.size(); ++i) {
        const Launch& L = launches[i];
        const std::vector<Arg>& a = L.a;
        auto V = [&](int k) -> const dh_view* { return a[k].count ? a[k].views.data() : nullptr; };
        auto F = [&](int k) -> float* { return (float*)(uintptr_t)a[k].p; };
        auto I = [&](int k) -> int { return (int)a[k].i; };
        int rc;
        switch (L.entry) {
        case E_CONV:
            rc = dh_conv2d_f32(ctx, V(0), F(1), a[2].count ? &a[2].packed : nullptr, &a[3].desc, V(4), stream);
            break;
        case E_SEPCONV:
            rc = dh_sepconv2d_f32(ctx, V(0), F(1), F(2), a[3].count ? &a[3].packed : nullptr, &a[4].desc, V(5), stream);
            break;
        case E_MAXPOOL: rc = dh_maxpool2d_f32(ctx, V(0), I(1), I(2), I(3), I(4), I(5), V(6), stream); break;
        case E_UPSAMPLE_ADD: rc = dh_upsample2x_add_f32(ctx, V(0), V(1), V(2), stream); break;
        case E_ADD_N: rc = dh_add_n_f32(ctx, V(0), I(1), F(2), F(3), I(4), V(5), stream); break;
        case E_SAM2D: rc = dh_softargmax2d_f32(ctx, V(0), V(1), a[2].f, I(3), F(4), F(5), V(6), stream); break;
        case E_SAM2D_CTX: rc = dh_softargmax2d_ctx_f32(ctx, V(0), I(1), I(2), a[3].f, F(4), F(5), stream); break;
        case E_SAM3D: rc = dh_softargmax3d_f32(ctx, V(0), I(1), I(2), F(3), F(4), stream); break;
        case E_SAM3D_EX: rc = dh_softargmax3d_ex_f32(ctx, V(0), I(1), I(2), a[3].f, F(4), F(5), V(6), stream); break;
        case E_KRON: rc = dh_kron_pool_f32(ctx, V(0), V(1), F(2), stream); break;
        case E_ZEROPAD: rc = dh_zeropad2d_f32(ctx, V(0), I(1), I(2), V(3), stream); break;
        case E_MAXMIN_POOL: rc = dh_maxmin_pool2d_f32(ctx, V(0), V(1), stream); break;
        case E_GLOBAL_MAXMIN_SOFTMAX: rc = dh_global_maxmin_softmax_f32(ctx, V(0), F(1), stream); break;
        default: rc = dh_mask_mul_f32(ctx, F(0), F(1), a[2].i, I(3), F(4), stream); break;
        }
        if (rc) {
            char msg[512];
            snprintf(msg, sizeof(msg), "%s", dh_last_error());
            dh_set_error("%s %zu (%s): %s", what, i, L.label.c_str(), msg);
            return rc;
        }
    }
    return 0;
}

// A model file's launch list, input and outputs at batch n (1 <= n <= N, the exported one; version 2): every view into
// an activation slot and dh_mask_mul_f32's rows over one scale by n / N, which check_items made exact, and each
// output's shape[0] becomes n.  Pointers stay file references: only item counts change.
void rebatch(const Parsed& m, int n, std::vector<Launch>* launches, dh_view* input, std::vector<Output>* outputs) {
    const int64_t N = m.info.clip_items;
    auto scale = [&](dh_view& v) {
        if (v.p && ref_arena(v.p) >= kArenaSlot0) v.n = (int32_t)(v.n / N * n);
    };
    scale(*input);
    for (Output& o : *outputs) {
        scale(o.view);
        o.info.shape[0] = n;
    }
    for (Launch& L : *launches) {
        for (Arg& a : L.a) {
            for (dh_view& v : a.views) scale(v);
            if (a.tag == 'd' && a.count) {
                scale(a.desc.res[0]);
                scale(a.desc.res[1]);
                scale(a.desc.pool_out);
            }
        }
        if (L.entry == E_MASK_MUL && ref_arena((void*)(uintptr_t)L.a[0].p) >= kArenaSlot0)
            L.a[2].i = L.a[2].i / N * n;
    }
}

// synchronise ctx's device, then free `dev`
cudaError_t free_device(dh_ctx* ctx, void* dev) {
    if (!dev) return cudaSuccess;
    int prev = 0;
    cudaGetDevice(&prev);
    cudaSetDevice(ctx->device);
    cudaError_t e = cudaDeviceSynchronize();            // no launch may still read the memory
    cudaError_t f = cudaFree(dev);
    if (e == cudaSuccess) e = f;
    cudaSetDevice(prev);
    return e;
}

}  // namespace

struct dh_model {
    dh_ctx* ctx;
    void* dev;
    Parsed m;                         // as read: pointers are file references, item counts the exported batch's
    Relocator R;
    void* workspace;
    int batch;                        // what forwards run at: the launches, input and outputs below
    std::vector<Launch> launches;     // relocated and planned
    dh_view input;
    std::vector<Output> outputs;
};

// Bind M at batch n: rewrite, relocate and plan a copy of the file's launch list, and only if every convolution has a
// kernel within the file's workspace make it the one forwards issue.  Host-only: nothing is launched.
static int bind_batch(dh_model* M, int n, const char* what) {
    std::vector<Launch> launches = M->m.launches;
    dh_view input = M->m.input;
    std::vector<Output> outputs = M->m.outputs;
    if (n != M->m.info.clip_items) rebatch(M->m, n, &launches, &input, &outputs);
    M->R.fix(input);
    for (Output& o : outputs) M->R.fix(o.view);
    TRY(relocate_and_plan(M->ctx, M->R, &launches, M->m.info.workspace_bytes, what));
    M->launches.swap(launches);
    M->input = input;
    M->outputs.swap(outputs);
    M->batch = n;
    return 0;
}

extern "C" int dh_model_inspect(const char* path, dh_model_info* info, int64_t* slot_bytes, int max_slots,
                                dh_model_output_info* outputs, int max_outputs) {
    DH_CHECK_ARG(info != nullptr, "dh_model_inspect: info is NULL");
    Parsed m;
    TRY(parse_file(path, &m));
    *info = m.info;
    for (int s = 0; slot_bytes && s < max_slots && s < m.info.n_slots; ++s) slot_bytes[s] = m.arena_bytes[kArenaSlot0 + s];
    for (int k = 0; outputs && k < max_outputs && k < m.info.n_outputs; ++k) outputs[k] = m.outputs[k].info;
    return 0;
}

extern "C" int dh_model_load(dh_ctx* ctx, const char* path, dh_model** out) {
    DH_CHECK_ARG(ctx && out, "dh_model_load: NULL ctx or out");
    *out = nullptr;
    dh_model* M = new dh_model();
    M->ctx = ctx;
    M->dev = nullptr;
    int rc = parse_file(path, &M->m);
    if (rc) { delete M; return rc; }
    Parsed& m = M->m;
    rc = upload(ctx, "dh_model_load", m.info.device_bytes, m.arena_bytes, m.weights, m.packed, &M->dev, &M->R);
    if (rc) { delete M; return rc; }
    M->workspace = M->R.base[kArenaWorkspace];
    // the host copies of the weights are on the device now
    std::vector<uint8_t>().swap(m.weights);
    std::vector<uint8_t>().swap(m.packed);
    rc = bind_batch(M, m.info.clip_items, "dh_model_load: launch");
    if (rc) {
        cudaFree(M->dev);
        delete M;
        return rc;
    }
    *out = M;
    return 0;
}

extern "C" int dh_model_set_batch(dh_model* M, int n) {
    DH_CHECK_ARG(M, "dh_model_set_batch: model is NULL");
    const int N = M->m.info.clip_items;
    DH_CHECK_ARG(n >= 1 && n <= N, "dh_model_set_batch: n = %d is outside [1, %d], the batch the file was exported at",
                 n, N);
    DH_CHECK_ARG(!M->m.slot_kind.empty() || n == N,
                 "dh_model_set_batch: the file is format version %d, which runs at its exported batch %d only; "
                 "export the model again (Model.export) to run it at n = %d", M->m.info.version, N, n);
    if (n == M->batch) return 0;
    return bind_batch(M, n, "dh_model_set_batch: launch");
}

extern "C" int dh_model_batch(const dh_model* M) {
    DH_CHECK_ARG(M, "dh_model_batch: model is NULL");
    return M->batch;
}

extern "C" int dh_model_input(const dh_model* M, dh_view* view) {
    DH_CHECK_ARG(M && view, "dh_model_input: NULL argument");
    *view = M->input;
    return 0;
}

extern "C" int dh_model_output(const dh_model* M, int k, dh_view* view, dh_model_output_info* info) {
    DH_CHECK_ARG(M, "dh_model_output: model is NULL");
    DH_CHECK_ARG(k >= 0 && k < M->m.info.n_outputs, "dh_model_output: output %d of %d", k, M->m.info.n_outputs);
    if (view) *view = M->outputs[k].view;
    if (info) *info = M->outputs[k].info;
    return 0;
}

extern "C" int dh_model_forward(dh_model* M, void* stream) {
    DH_CHECK_ARG(M, "dh_model_forward: model is NULL");
    return issue(M->ctx, M->launches, M->workspace, M->m.info.workspace_bytes, stream, "dh_model_forward: launch");
}

extern "C" int dh_model_free(dh_model* M) {
    if (!M) return 0;
    cudaError_t e = free_device(M->ctx, M->dev);
    delete M;
    if (e != cudaSuccess) {
        dh_set_error("dh_model_free: %s", cudaGetErrorString(e));
        return (int)e;
    }
    return 0;
}

// ---- live video: ClipStream.export files ------------------------------------------------------------------------------
struct dh_stream {
    dh_ctx* ctx;
    void* dev;
    StreamParsed m;
    void *ws_frame, *ws_clip;
    dh_clip_window* table;        // device: the boundary table of dh_clip_window_f32
    dh_view* outs;                // device: the clip-output views of dh_stream_ready_f32
    int32_t *counter, *counts, *ready;
};

extern "C" int dh_stream_inspect(const char* path, dh_stream_info* info, dh_model_output_info* outputs, int max_outputs) {
    DH_CHECK_ARG(info != nullptr, "dh_stream_inspect: info is NULL");
    StreamParsed m;
    TRY(parse_stream_file(path, &m));
    *info = m.info;
    for (int k = 0; outputs && k < max_outputs && k < (int)m.outputs.size(); ++k) outputs[k] = m.outputs[k].info;
    return 0;
}

extern "C" int dh_stream_load(dh_ctx* ctx, const char* path, dh_stream** out) {
    DH_CHECK_ARG(ctx && out, "dh_stream_load: NULL ctx or out");
    *out = nullptr;
    dh_stream* st = new dh_stream();
    st->ctx = ctx;
    int rc = parse_stream_file(path, &st->m);
    if (rc) { delete st; return rc; }
    StreamParsed& m = st->m;
    const dh_stream_info& I = m.info;
    Relocator R;
    rc = upload(ctx, "dh_stream_load", I.device_bytes, m.arena_bytes, m.weights, m.packed, &st->dev, &R);
    if (rc) { delete st; return rc; }
    std::vector<uint8_t>().swap(m.weights);
    std::vector<uint8_t>().swap(m.packed);
    st->ws_frame = R.base[kArenaWorkspace];
    st->ws_clip = R.base[kArenaClipWorkspace];
    int64_t base = 0;
    for (int64_t b : m.arena_bytes) base += (b + kArenaAlign - 1) / kArenaAlign * kArenaAlign;
    const StreamTail tail = stream_tail(base, I.n_boundary, I.n_clip_outputs, I.n_streams);
    uint8_t* dev = (uint8_t*)st->dev;
    st->table = (dh_clip_window*)(dev + tail.table);
    st->outs = (dh_view*)(dev + tail.outs);
    st->counter = (int32_t*)(dev + tail.counter);
    st->counts = (int32_t*)(dev + tail.counts);
    st->ready = (int32_t*)(dev + tail.ready);
    R.fix(m.input);
    for (Output& o : m.outputs) R.fix(o.view);
    for (dh_clip_window& e : m.boundary) {
        R.fix(e.src);
        R.fix(e.dst);
        R.fix(e.ring);
    }
    std::vector<dh_view> clip_views;
    for (int k = I.n_frame_outputs; k < (int)m.outputs.size(); ++k) clip_views.push_back(m.outputs[k].view);
    int prev = 0;
    cudaGetDevice(&prev);
    cudaError_t e = cudaSetDevice(ctx->device);
    if (e == cudaSuccess)
        e = cudaMemcpy(st->table, m.boundary.data(), m.boundary.size() * sizeof(dh_clip_window), cudaMemcpyHostToDevice);
    if (e == cudaSuccess)
        e = cudaMemcpy(st->outs, clip_views.data(), clip_views.size() * sizeof(dh_view), cudaMemcpyHostToDevice);
    cudaSetDevice(prev);
    if (e != cudaSuccess) {
        dh_set_error("dh_stream_load: %s", cudaGetErrorString(e));
        rc = (int)e;
    }
    if (!rc) rc = relocate_and_plan(ctx, R, &m.frame, I.frame_workspace_bytes, "dh_stream_load: frame launch");
    if (!rc) rc = relocate_and_plan(ctx, R, &m.clip, I.clip_workspace_bytes, "dh_stream_load: clip launch");
    if (rc) {
        cudaFree(st->dev);
        delete st;
        return rc;
    }
    *out = st;
    return 0;
}

extern "C" int dh_stream_input(const dh_stream* st, dh_view* view) {
    DH_CHECK_ARG(st && view, "dh_stream_input: NULL argument");
    *view = st->m.input;
    return 0;
}

extern "C" int dh_stream_push(dh_stream* st, void* stream) {
    DH_CHECK_ARG(st, "dh_stream_push: stream is NULL");
    const dh_stream_info& I = st->m.info;
    TRY(issue(st->ctx, st->m.frame, st->ws_frame, I.frame_workspace_bytes, stream, "dh_stream_push: frame launch"));
    TRY(dh_clip_window_f32(st->ctx, st->table, I.n_boundary, I.n_streams, I.frames_per_clip, st->counter, stream));
    TRY(issue(st->ctx, st->m.clip, st->ws_clip, I.clip_workspace_bytes, stream, "dh_stream_push: clip launch"));
    return dh_stream_ready_f32(st->ctx, st->counts, I.n_streams, I.frames_per_clip, st->outs, I.n_clip_outputs,
                               st->ready, stream);
}

extern "C" int dh_stream_reset(dh_stream* st, const int32_t* ids, int n, void* stream) {
    DH_CHECK_ARG(st, "dh_stream_reset: stream is NULL");
    const int S = st->m.info.n_streams;
    DH_CHECK_ARG(ids == nullptr || n >= 0, "dh_stream_reset: n = %d", n);
    for (int i = 0; ids && i < n; ++i)
        DH_CHECK_ARG(ids[i] >= 0 && ids[i] < S, "dh_stream_reset: id %d is outside [0, %d)", ids[i], S);
    int prev = 0;
    cudaGetDevice(&prev);
    cudaError_t e = cudaSetDevice(st->ctx->device);
    if (!ids) {
        if (e == cudaSuccess) e = cudaMemsetAsync(st->counts, 0, (size_t)S * sizeof(int32_t), (cudaStream_t)stream);
    } else {
        for (int i = 0; i < n && e == cudaSuccess; ++i)
            e = cudaMemsetAsync(st->counts + ids[i], 0, sizeof(int32_t), (cudaStream_t)stream);
    }
    cudaSetDevice(prev);
    if (e != cudaSuccess) {
        dh_set_error("dh_stream_reset: %s", cudaGetErrorString(e));
        return (int)e;
    }
    return 0;
}

extern "C" int dh_stream_output(const dh_stream* st, int k, dh_view* view, dh_model_output_info* info) {
    DH_CHECK_ARG(st, "dh_stream_output: stream is NULL");
    const int n = (int)st->m.outputs.size();
    DH_CHECK_ARG(k >= 0 && k < n, "dh_stream_output: output %d of %d", k, n);
    if (view) *view = st->m.outputs[k].view;
    if (info) *info = st->m.outputs[k].info;
    return 0;
}

extern "C" int dh_stream_ready(const dh_stream* st, const int32_t** ready_dev) {
    DH_CHECK_ARG(st && ready_dev, "dh_stream_ready: NULL argument");
    *ready_dev = st->ready;
    return 0;
}

extern "C" int dh_stream_free(dh_stream* st) {
    if (!st) return 0;
    cudaError_t e = free_device(st->ctx, st->dev);
    delete st;
    if (e != cudaSuccess) {
        dh_set_error("dh_stream_free: %s", cudaGetErrorString(e));
        return (int)e;
    }
    return 0;
}
