// Baseline JPEG decoding on the GPU, bit-identical to Pillow's Image.open(...).convert('RGB') (libjpeg-turbo in its
// default configuration), for the files deephar_b200/jpeg.py routes here.  Three stages, each a launch:
//   1. entropy decoding: one thread per restart interval (per image without restart markers) -- 0xFF00 unstuffing,
//      canonical Huffman decoding through a 9-bit table plus a per-length search, DC prediction reset at each
//      interval, sign extension -> int16 coefficients in natural order;
//   2. dequantisation + the ISLOW integer IDCT + level shift + range limit: one thread per 8x8 block -> sample planes;
//   3. fancy upsampling of the chroma (h2v1, h2v2, libjpeg's rounding biases, edge columns and context rows
//      replicated) + integer YCbCr -> RGB (SCALEBITS 16): one thread per pixel -> packed RGB.
// Anything the files do that libjpeg would only warn about (a bad code, an interval that runs out of data, a run
// past coefficient 63) and IDCT values outside the range where libjpeg-turbo's C and SIMD IDCTs agree set the image's
// status word; the host re-decodes those images with Pillow.  oracle/jpeg.py is the model these kernels port.
#include "common.cuh"

namespace {

__constant__ uint8_t kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                    12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                    35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                    58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// ---- stage 1: entropy decoding ----------------------------------------------------------------------------------

struct BitReader {
    const uint8_t* p;
    const uint8_t* end;
    uint64_t buf;   // next bits, MSB first
    int n;          // valid bits in buf
    int zeros;      // zero bits fed after the segment's last byte
};

// Top up to at least 57 bits.  Reads stay inside [p, end): the host cuts segments at markers, strips fill bytes and
// routes files with 0xFF 0xFF inside a segment to Pillow, so every 0xFF read here is followed by its stuffed 0x00.
__device__ __forceinline__ void fill(BitReader& r) {
    while (r.n <= 56) {
        uint32_t byte = 0;
        if (r.p < r.end) {
            byte = *r.p;
            r.p += byte == 0xFF ? 2 : 1;
        } else {
            r.zeros += 8;
        }
        r.buf |= (uint64_t)byte << (56 - r.n);
        r.n += 8;
    }
}

__device__ __forceinline__ int decode_symbol(BitReader& r, const dh_jpeg_huff* __restrict__ t, int& err) {
    fill(r);
    const uint32_t e = t->lut[r.buf >> 55];
    if (e) {
        const int len = e >> 8;
        r.buf <<= len;
        r.n -= len;
        return e & 0xFF;
    }
    const int c16 = (int)(r.buf >> 48);
    for (int len = 10; len <= 16; ++len) {
        const int code = c16 >> (16 - len);
        if (code <= t->maxcode[len]) {
            r.buf <<= len;
            r.n -= len;
            return t->vals[(code + t->valoff[len]) & 0xFF];
        }
    }
    err |= DH_JPEG_BAD_CODE;
    return 0;
}

// s in 1..15 additional bits after a symbol (decode_symbol left >= 41 bits), sign-extended (HUFF_EXTEND)
__device__ __forceinline__ int receive_extend(BitReader& r, int s) {
    const int v = (int)(r.buf >> (64 - s));
    r.buf <<= s;
    r.n -= s;
    return v < (1 << (s - 1)) ? v - (1 << s) + 1 : v;
}

__global__ void jpeg_entropy_kernel(const dh_jpeg_batch b) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= b.n_segments) return;
    const dh_jpeg_segment seg = b.segments[s];
    const dh_jpeg_image& im = b.images[seg.image];
    BitReader r{b.data + seg.begin, b.data + seg.end, 0, 0, 0};
    int pred[3] = {0, 0, 0};
    int err = 0;
    const int nc = im.ncomp, mcus_x = im.mcus_x;
    for (int m = seg.mcu0; m < seg.mcu0 + seg.mcus && !err; ++m) {
        const int my = m / mcus_x, mx = m - my * mcus_x;
        for (int c = 0; c < nc && !err; ++c) {
            const int hs = c == 0 ? im.hs : 1, vs = c == 0 ? im.vs : 1;
            const dh_jpeg_huff* dct = b.huff + im.dc[c];
            const dh_jpeg_huff* act = b.huff + im.ac[c];
            for (int v = 0; v < vs; ++v) {
                for (int u = 0; u < hs; ++u) {
                    int16_t* blk = b.coef + im.coef[c] + ((int64_t)(my * vs + v) * im.bw[c] + mx * hs + u) * 64;
                    const int t = decode_symbol(r, dct, err);
                    if (t) pred[c] += receive_extend(r, t);
                    if (pred[c] < -32768 || pred[c] > 32767) err |= DH_JPEG_BAD_INDEX;
                    blk[0] = (int16_t)pred[c];
                    for (int k = 1; k < 64;) {
                        const int rs = decode_symbol(r, act, err);
                        const int run = rs >> 4, size = rs & 15;
                        if (size) {
                            k += run;
                            if (k > 63) {
                                err |= DH_JPEG_BAD_INDEX;
                                break;
                            }
                            blk[kZigzag[k]] = (int16_t)receive_extend(r, size);
                            ++k;
                        } else if (run == 15) {
                            k += 16;                                   // ZRL
                        } else {
                            break;                                     // EOB
                        }
                    }
                }
            }
        }
    }
    if (r.zeros > r.n) err |= DH_JPEG_NO_DATA;                        // bits were taken past the segment's end
    if (err) atomicOr(b.status + seg.image, err);
}

// ---- stage 2: dequantisation + ISLOW IDCT ----------------------------------------------------------------------

constexpr int CONST_BITS = 13, PASS1_BITS = 2;
// libjpeg-turbo's IDCT runs as C (int arithmetic, a wrapping range-limit table) or as SIMD code (16-bit dequantised
// values and workspace, saturating packs).  Both give the same samples while every dequantised coefficient and
// workspace value stays within +-AGREE and every output within [-512, 511] (there the table is a plain clamp);
// oracle/jpeg.py states the same rule.  Encoded 8-bit images stay far inside it.
constexpr int AGREE = 8191;

__device__ __forceinline__ int64_t descale(int64_t x, int n) { return (x + ((int64_t)1 << (n - 1))) >> n; }

// one 1-D pass of jidctint.c's butterfly on in[0..7] (stride 1) -> out[0..7] before descaling
__device__ __forceinline__ void idct_1d(const int64_t d[8], int64_t o[8]) {
    int64_t z1 = (d[2] + d[6]) * 4433;
    const int64_t tmp2 = z1 + d[6] * -15137, tmp3 = z1 + d[2] * 6270;
    const int64_t tmp0 = (d[0] + d[4]) * 8192, tmp1 = (d[0] - d[4]) * 8192;
    const int64_t t10 = tmp0 + tmp3, t13 = tmp0 - tmp3, t11 = tmp1 + tmp2, t12 = tmp1 - tmp2;
    int64_t o0 = d[7], o1 = d[5], o2 = d[3], o3 = d[1];
    z1 = o0 + o3;
    int64_t z2 = o1 + o2, z3 = o0 + o2, z4 = o1 + o3;
    const int64_t z5 = (z3 + z4) * 9633;
    o0 *= 2446;
    o1 *= 16819;
    o2 *= 25172;
    o3 *= 12299;
    z1 *= -7373;
    z2 *= -20995;
    z3 = z3 * -16069 + z5;
    z4 = z4 * -3196 + z5;
    o0 += z1 + z3;
    o1 += z2 + z4;
    o2 += z2 + z3;
    o3 += z1 + z4;
    o[0] = t10 + o3; o[7] = t10 - o3;
    o[1] = t11 + o2; o[6] = t11 - o2;
    o[2] = t12 + o1; o[5] = t12 - o1;
    o[3] = t13 + o0; o[4] = t13 - o0;
}

__global__ void __launch_bounds__(128) jpeg_idct_kernel(const dh_jpeg_batch b) {
    const dh_jpeg_image& im = b.images[blockIdx.y];
    int blk = blockIdx.x * blockDim.x + threadIdx.x;
    if (blk >= im.nblocks) return;
    int c = 0;
    while (c + 1 < im.ncomp && blk >= im.bw[c] * im.bh[c]) blk -= im.bw[c] * im.bh[c], ++c;
    const int bw = im.bw[c], by = blk / bw, bx = blk - by * bw;
    const int4* src = reinterpret_cast<const int4*>(b.coef + im.coef[c] + (int64_t)blk * 64);
    const uint16_t* q = b.qtab + (int64_t)im.qt[c] * 64;
    int ws[64];
    bool ok = true;
#pragma unroll
    for (int v = 0; v < 8; ++v) {                                     // dequantise: 8 coefficients per 16-byte load
        const int4 raw = src[v];
        const int16_t* c8 = reinterpret_cast<const int16_t*>(&raw);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            ws[v * 8 + k] = (int)c8[k] * (int)q[v * 8 + k];
            ok &= ws[v * 8 + k] >= -AGREE && ws[v * 8 + k] <= AGREE;
        }
    }
#pragma unroll
    for (int col = 0; col < 8; ++col) {                               // pass 1: columns, in place
        int64_t d[8], o[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) d[k] = ws[k * 8 + col];
        idct_1d(d, o);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int64_t w = descale(o[k], CONST_BITS - PASS1_BITS);
            ok &= w >= -AGREE && w <= AGREE;
            ws[k * 8 + col] = (int)w;
        }
    }
    uint8_t* dst = b.planes + im.plane[c] + (int64_t)by * 8 * (bw * 8) + bx * 8;
#pragma unroll
    for (int row = 0; row < 8; ++row) {                               // pass 2: rows -> samples
        int64_t d[8], o[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) d[k] = ws[row * 8 + k];
        idct_1d(d, o);
        uint32_t lo = 0, hi = 0;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int x = (int)descale(o[k], CONST_BITS + PASS1_BITS + 3);
            ok &= x >= -512 && x <= 511;
            const uint32_t px = (uint32_t)min(max(x + 128, 0), 255);
            if (k < 4) lo |= px << (8 * k); else hi |= px << (8 * (k - 4));
        }
        *reinterpret_cast<uint2*>(dst + (int64_t)row * bw * 8) = make_uint2(lo, hi);
    }
    if (!ok) atomicOr(b.status + blockIdx.y, DH_JPEG_RANGE);
}

// ---- stage 3: upsampling + colour conversion -------------------------------------------------------------------

// chroma sample at full-resolution (x, y): plane P (pitch bytes per row), cw x ch valid samples
__device__ __forceinline__ int chroma(const uint8_t* __restrict__ P, int pitch, int x, int y, int hs, int vs, int cw,
                                      int ch) {
    if (hs == 1) return P[(int64_t)y * pitch + x];                     // 4:4:4
    const int i = x >> 1;
    if (cw <= 2) return P[(int64_t)(y >> (vs - 1)) * pitch + i];       // libjpeg replicates planes this narrow
    const int nb = (x & 1) ? min(i + 1, cw - 1) : max(i - 1, 0);
    if (vs == 1) {                                                     // h2v1: 3/4 nearer + 1/4 further
        const uint8_t* row = P + (int64_t)y * pitch;
        return (3 * row[i] + row[nb] + 1 + (x & 1)) >> 2;
    }
    const int j = y >> 1;                                              // h2v2: column sums of the nearer and further row
    const int far = (y & 1) ? min(j + 1, ch - 1) : max(j - 1, 0);
    const uint8_t* r0 = P + (int64_t)j * pitch;
    const uint8_t* r1 = P + (int64_t)far * pitch;
    const int s0 = 3 * r0[i] + r1[i], s1 = 3 * r0[nb] + r1[nb];
    return (3 * s0 + s1 + 8 - (x & 1)) >> 4;
}

__global__ void jpeg_color_kernel(const dh_jpeg_batch b) {
    const dh_jpeg_image& im = b.images[blockIdx.z];
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    const int w = im.w, h = im.h;
    if (x >= w || y >= h) return;
    const int Y = b.planes[im.plane[0] + (int64_t)y * im.bw[0] * 8 + x];
    uint8_t* o = b.out + im.out + ((int64_t)y * w + x) * 3;
    if (im.ncomp == 1) {
        o[0] = o[1] = o[2] = (uint8_t)Y;
        return;
    }
    const int hs = im.hs, vs = im.vs, cw = (w + hs - 1) / hs, ch = (h + vs - 1) / vs;
    const int cb = chroma(b.planes + im.plane[1], im.bw[1] * 8, x, y, hs, vs, cw, ch) - 128;
    const int cr = chroma(b.planes + im.plane[2], im.bw[2] * 8, x, y, hs, vs, cw, ch) - 128;
    const int r = Y + ((91881 * cr + 32768) >> 16);                    // jdcolor.c: FIX(1.40200) ...
    const int g = Y + ((-22554 * cb - 46802 * cr + 32768) >> 16);      // FIX(0.34414), FIX(0.71414)
    const int bl = Y + ((116130 * cb + 32768) >> 16);                  // FIX(1.77200)
    o[0] = (uint8_t)min(max(r, 0), 255);
    o[1] = (uint8_t)min(max(g, 0), 255);
    o[2] = (uint8_t)min(max(bl, 0), 255);
}

}  // namespace

extern "C" int dh_jpeg_decode(dh_ctx* ctx, const dh_jpeg_batch* batch, int stages, void* stream) {
    DH_CHECK_ARG(ctx && batch, "dh_jpeg_decode: NULL argument");
    const dh_jpeg_batch b = *batch;
    DH_CHECK_ARG(b.n_images >= 0 && b.n_images <= 65535 && b.n_segments >= 0, "dh_jpeg_decode: at most 65535 images");
    DH_CHECK_ARG(stages >= 0 && stages <= 7, "dh_jpeg_decode: stages is a mask of 1 | 2 | 4");
    if (b.n_images == 0) return 0;
    DH_CHECK_ARG(b.images && b.status, "dh_jpeg_decode: NULL table");
    DH_CHECK_ARG(!(stages & 1) || (b.segments && b.huff && b.data && b.coef && b.coef_elems >= 0),
                 "dh_jpeg_decode: entropy stage needs segments, tables, data and coefficients");
    DH_CHECK_ARG(!(stages & 2) || (b.coef && b.qtab && b.planes && b.max_blocks >= 0), "dh_jpeg_decode: IDCT stage needs coefficients, tables and planes");
    DH_CHECK_ARG(!(stages & 4) || (b.planes && b.out && b.max_h >= 0 && b.max_w >= 0), "dh_jpeg_decode: colour stage needs planes and output");
    cudaStream_t s = (cudaStream_t)stream;
    int launches = 0;
    if (stages & 1) {
        cudaMemsetAsync(b.coef, 0, b.coef_elems * sizeof(int16_t), s);
        cudaMemsetAsync(b.status, 0, b.n_images * sizeof(int32_t), s);
        // each thread decodes serially: spread the segments over every SM sub-partition before packing warps
        int tpb = 1;
        while (tpb < 32 && (int64_t)tpb * 4 * ctx->num_sms < b.n_segments) tpb *= 2;
        if (b.n_segments > 0) {
            jpeg_entropy_kernel<<<(b.n_segments + tpb - 1) / tpb, tpb, 0, s>>>(b);
            ++launches;
        }
    }
    if ((stages & 2) && b.max_blocks > 0) {
        jpeg_idct_kernel<<<dim3((b.max_blocks + 127) / 128, b.n_images), 128, 0, s>>>(b);
        ++launches;
    }
    if ((stages & 4) && b.max_h > 0 && b.max_w > 0) {
        jpeg_color_kernel<<<dim3((b.max_w + 31) / 32, (b.max_h + 7) / 8, b.n_images), dim3(32, 8), 0, s>>>(b);
        ++launches;
    }
    DH_LAUNCH_EPILOGUE(ctx, launches);
}
