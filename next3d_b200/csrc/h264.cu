// H.264 encoder (Constrained Baseline, CAVLC) for the video writer (next3d_b200/video.py; DESIGN.md section 3.5).
//
// One slice per macroblock (MB) row, so every neighbour above an MB is in another slice and "not available": intra 16x16 uses DC
// or horizontal prediction, the P_Skip MV is (0,0), and the MV predictor is the left MB's MV.  Rows are independent.
//   h264_rgb_to_yuv   uint8 RGB HWC -> padded I420 planes, BT.601 limited range in integers.
//   h264_intra_rows   IDR frames: one warp per MB row, MBs in order (each needs its left neighbour's reconstruction); lanes 0-15
//                     own the luma 4x4 blocks, lanes 16-23 the chroma blocks.
//   h264_inter_mbs    P frames: one block per MB; integer-pel full search over [-kSearch, kSearch]^2 against the previous
//                     reconstruction (coordinates clamped, as the decoder clamps them), then transform / quantise / reconstruct.
//   h264_write_rows   CAVLC: one thread per row writes the slice NAL unit (header, MB layer, trailing bits, emulation prevention)
//                     into its own bounded slot, length-prefixed.
//   h264_pack         concatenates the slots into one AVCC sample (an MP4 sample of the frame).
// The rate-controlled stream (n3d_h264_encode_rc) runs the same kernels with kRc = true: every kernel reads the picture's QP from
// the controller state, h264_inter_mbs refines the vector to quarter samples, and two kernels are added:
//   h264_deblock      in-loop deblocking (8.7) in place on the reconstruction: one warp per MB row, rows taken in order through an
//                     atomic ticket, MB x of a row waiting until the row above has finished MB x + 1 (the standard's raster order).
//   h264_rc_update    one thread: the frame's size -> the controller state and the next picture's QP.
// The numpy restatement in tests/h264_oracle.py (Encoder, RcEncoder: kRc false, true) makes the same decisions and writes the
// same bytes.
#include "common.cuh"

namespace {

constexpr int kSearch = 16;                     // integer-pel search range (luma samples); MVs are stored in quarter-pel units
constexpr int kWin = 16 + 2 * kSearch;          // reference window side
constexpr int kCands = (2 * kSearch + 1) * (2 * kSearch + 1);
constexpr int kLevelMax = 2063;                 // largest |level| CAVLC codes with level_prefix <= 15 (Baseline) at any suffixLength
constexpr int kMaxFs = 139264;                  // level 6.2 MaxFS (macroblocks)
constexpr int kBlockBits = 16 + 3 + 16 * 28 + 9 + 15 * 11;   // coeff_token, T1 signs, 16 escaped levels, total_zeros, run_before
constexpr int kMbBits = 27 * kBlockBits + 128;  // 27 residual blocks + MB header (skip run, type, mvd, cbp, qp delta)
constexpr int kMvOff = 128;                     // key offset of quarter-sample vector components (|mv| <= 4 * kSearch + 3)
constexpr int kPat = 22;                        // quarter-sample patch side: the 16 samples +- 1 of refinement, 2 + 3 filter taps
constexpr uint32_t kSpinLimit = 1u << 24;       // bounded waits of h264_deblock (~1 s of __nanosleep(64)), then trap

// Rate-control state (int64 fields, N3D_H264_RC_STATE_BYTES).  Fullness: the stream's excess over bitrate x time, in 1/fps_num bits.
enum { kRcBitrate, kRcNum, kRcDen, kRcQpMin, kRcQpMax, kRcQp, kRcFullness, kRcFrames, kRcPrevIdr, kRcFields = 16 };
static_assert(kRcFields * 8 == N3D_H264_RC_STATE_BYTES, "rate-control state size");

// Per-MB record between the decision kernels and the writer.  lv: levels in zig-zag order per block: 0-15 luma 4x4 blocks
// (luma4x4BlkIdx order; index 0 unused for I_16x16), 16 luma DC (I_16x16), 17 chroma DC (Cb 0-3, Cr 4-7), 18-21 Cb AC, 22-25 Cr AC
// (index 0 unused).  Unused entries are zero.
struct MbRec {
    int16_t lv[26][16];
    int32_t mode;          // I: Intra16x16PredMode (1 horizontal, 2 DC); P: 0
    int32_t mvx, mvy;      // quarter-pel (P)
    int32_t pad;
};

__constant__ int8_t c_zz[16] = {0, 1, 4, 8, 5, 2, 3, 6, 9, 12, 13, 10, 7, 11, 14, 15};
__constant__ int8_t c_blk_x[16] = {0, 1, 0, 1, 2, 3, 2, 3, 0, 1, 0, 1, 2, 3, 2, 3};
__constant__ int8_t c_blk_y[16] = {0, 0, 1, 1, 0, 0, 1, 1, 2, 2, 3, 3, 2, 2, 3, 3};
__constant__ uint8_t c_lambda[52] = {0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 4, 4, 5, 5, 6, 7, 7, 8, 9,
                                     10, 12, 13, 15, 17, 19, 21, 23, 26, 30, 33, 37, 42, 47, 53, 59, 66, 74, 83};
__constant__ int c_mf[6][3] = {{13107, 5243, 8066}, {11916, 4660, 7490}, {10082, 4194, 6554}, {9362, 3647, 5825}, {8192, 3355, 5243}, {7282, 2893, 4559}};
__constant__ int c_v[6][3] = {{10, 16, 13}, {11, 18, 14}, {13, 20, 16}, {14, 23, 18}, {16, 25, 20}, {18, 29, 23}};
__constant__ uint8_t c_qpc[52] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 19, 20, 21, 22, 23, 24, 25, 26, 27, 28,
                                  29, 29, 30, 31, 32, 32, 33, 34, 34, 35, 35, 36, 36, 37, 37, 37, 38, 38, 38, 39, 39, 39, 39};
// deblocking: alpha' and beta' (Table 8-16), tC0' for bS = 1, 2, 3 (Table 8-17), by indexA / indexB (= qPav: offsets 0)
__constant__ uint8_t c_alpha[52] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 4, 4, 5, 6, 7, 8, 9, 10, 12, 13, 15, 17, 20, 22, 25,
                                    28, 32, 36, 40, 45, 50, 56, 63, 71, 80, 90, 101, 113, 127, 144, 162, 182, 203, 226, 255, 255};
__constant__ uint8_t c_beta[52] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 6, 6, 7, 7, 8, 8, 9, 9,
                                   10, 10, 11, 11, 12, 12, 13, 13, 14, 14, 15, 15, 16, 16, 17, 17, 18, 18};
__constant__ uint8_t c_tc0[52][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}, {0, 0, 0}, {0, 0, 0}, {0, 0, 0}, {0, 0, 0}, {0, 0, 0}, {0, 0, 0},
                                     {0, 0, 0}, {0, 0, 0}, {0, 0, 0}, {0, 0, 0}, {0, 0, 0}, {0, 0, 0}, {0, 0, 0}, {0, 0, 0}, {0, 0, 1},
                                     {0, 0, 1}, {0, 0, 1}, {0, 0, 1}, {0, 1, 1}, {0, 1, 1}, {1, 1, 1}, {1, 1, 1}, {1, 1, 1}, {1, 1, 1},
                                     {1, 1, 2}, {1, 1, 2}, {1, 1, 2}, {1, 1, 2}, {1, 2, 3}, {1, 2, 3}, {2, 2, 3}, {2, 2, 4}, {2, 3, 4},
                                     {2, 3, 4}, {3, 3, 5}, {3, 4, 6}, {3, 4, 6}, {4, 5, 7}, {4, 5, 8}, {4, 6, 9}, {5, 7, 10}, {6, 8, 11},
                                     {6, 8, 13}, {7, 10, 14}, {8, 11, 16}, {9, 12, 18}, {10, 13, 20}, {11, 15, 23}, {13, 17, 25}};
__constant__ uint8_t c_inter_cbp_code[48] = {0, 2, 3, 7, 4, 8, 17, 13, 5, 18, 9, 14, 10, 15, 16, 11, 1, 32, 33, 36, 34, 37, 44, 40,
                                             35, 45, 38, 41, 39, 42, 43, 19, 6, 24, 25, 20, 26, 21, 46, 28, 27, 47, 22, 29, 23, 30, 31, 12};

// coeff_token (Table 9-5), index 4 * TotalCoeff + TrailingOnes: 0 <= nC < 2, 2 <= nC < 4, 4 <= nC < 8, 8 <= nC
__constant__ uint8_t c_ct_len[4][68] = {
    {1, 0, 0, 0, 6, 2, 0, 0, 8, 6, 3, 0, 9, 8, 7, 5, 10, 9, 8, 6, 11, 10, 9, 7, 13, 11, 10, 8, 13, 13, 11, 9, 13, 13, 13, 10,
     14, 14, 13, 11, 14, 14, 14, 13, 15, 15, 14, 14, 15, 15, 15, 14, 16, 15, 15, 15, 16, 16, 16, 15, 16, 16, 16, 16, 16, 16, 16, 16},
    {2, 0, 0, 0, 6, 2, 0, 0, 6, 5, 3, 0, 7, 6, 6, 4, 8, 6, 6, 4, 8, 7, 7, 5, 9, 8, 8, 6, 11, 9, 9, 6, 11, 11, 11, 7,
     12, 11, 11, 9, 12, 12, 12, 11, 12, 12, 12, 11, 13, 13, 13, 12, 13, 13, 13, 13, 13, 14, 13, 13, 14, 14, 14, 13, 14, 14, 14, 14},
    {4, 0, 0, 0, 6, 4, 0, 0, 6, 5, 4, 0, 6, 5, 5, 4, 7, 5, 5, 4, 7, 5, 5, 4, 7, 6, 6, 4, 7, 6, 6, 4, 8, 7, 7, 5,
     8, 8, 7, 6, 9, 8, 8, 7, 9, 9, 8, 8, 9, 9, 9, 8, 10, 9, 9, 9, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10},
    {6, 0, 0, 0, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6,
     6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6}};
__constant__ uint8_t c_ct_bits[4][68] = {
    {1, 0, 0, 0, 5, 1, 0, 0, 7, 4, 1, 0, 7, 6, 5, 3, 7, 6, 5, 3, 7, 6, 5, 4, 15, 6, 5, 4, 11, 14, 5, 4, 8, 10, 13, 4,
     15, 14, 9, 4, 11, 10, 13, 12, 15, 14, 9, 12, 11, 10, 13, 8, 15, 1, 9, 12, 11, 14, 13, 8, 7, 10, 9, 12, 4, 6, 5, 8},
    {3, 0, 0, 0, 11, 2, 0, 0, 7, 7, 3, 0, 7, 10, 9, 5, 7, 6, 5, 4, 4, 6, 5, 6, 7, 6, 5, 8, 15, 6, 5, 4, 11, 14, 13, 4,
     15, 10, 9, 4, 11, 14, 13, 12, 8, 10, 9, 8, 15, 14, 13, 12, 11, 10, 9, 12, 7, 11, 6, 8, 9, 8, 10, 1, 7, 6, 5, 4},
    {15, 0, 0, 0, 15, 14, 0, 0, 11, 15, 13, 0, 8, 12, 14, 12, 15, 10, 11, 11, 11, 8, 9, 10, 9, 14, 13, 9, 8, 10, 9, 8,
     15, 14, 13, 13, 11, 14, 10, 12, 15, 10, 13, 12, 11, 14, 9, 12, 8, 10, 13, 8, 13, 7, 9, 12, 9, 12, 11, 10, 5, 8, 7, 6,
     1, 4, 3, 2},
    {3, 0, 0, 0, 0, 1, 0, 0, 4, 5, 6, 0, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 19, 20, 21, 22, 23, 24, 25, 26, 27, 28, 29,
     30, 31, 32, 33, 34, 35, 36, 37, 38, 39, 40, 41, 42, 43, 44, 45, 46, 47, 48, 49, 50, 51, 52, 53, 54, 55, 56, 57, 58, 59,
     60, 61, 62, 63}};
__constant__ uint8_t c_cdc_ct_len[20] = {2, 0, 0, 0, 6, 1, 0, 0, 6, 6, 3, 0, 6, 7, 7, 6, 6, 8, 8, 7};
__constant__ uint8_t c_cdc_ct_bits[20] = {1, 0, 0, 0, 7, 1, 0, 0, 4, 6, 1, 0, 3, 3, 2, 5, 2, 3, 2, 0};
// total_zeros (Tables 9-7, 9-8), [TotalCoeff - 1][total_zeros]
__constant__ uint8_t c_tz_len[15][16] = {
    {1, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 9}, {3, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 6, 6, 6, 6}, {4, 3, 3, 3, 4, 4, 3, 3, 4, 5, 5, 6, 5, 6},
    {5, 3, 4, 4, 3, 3, 3, 4, 3, 4, 5, 5, 5}, {4, 4, 4, 3, 3, 3, 3, 3, 4, 5, 4, 5}, {6, 5, 3, 3, 3, 3, 3, 3, 4, 3, 6},
    {6, 5, 3, 3, 3, 2, 3, 4, 3, 6}, {6, 4, 5, 3, 2, 2, 3, 3, 6}, {6, 6, 4, 2, 2, 3, 2, 5}, {5, 5, 3, 2, 2, 2, 4}, {4, 4, 3, 3, 1, 3},
    {4, 4, 2, 1, 3}, {3, 3, 1, 2}, {2, 2, 1}, {1, 1}};
__constant__ uint8_t c_tz_bits[15][16] = {
    {1, 3, 2, 3, 2, 3, 2, 3, 2, 3, 2, 3, 2, 3, 2, 1}, {7, 6, 5, 4, 3, 5, 4, 3, 2, 3, 2, 3, 2, 1, 0}, {5, 7, 6, 5, 4, 3, 4, 3, 2, 3, 2, 1, 1, 0},
    {3, 7, 5, 4, 6, 5, 4, 3, 3, 2, 2, 1, 0}, {5, 4, 3, 7, 6, 5, 4, 3, 2, 1, 1, 0}, {1, 1, 7, 6, 5, 4, 3, 2, 1, 1, 0},
    {1, 1, 5, 4, 3, 3, 2, 1, 1, 0}, {1, 1, 1, 3, 3, 2, 2, 1, 0}, {1, 0, 1, 3, 2, 1, 1, 1}, {1, 0, 1, 3, 2, 1, 1}, {0, 1, 1, 2, 1, 3},
    {0, 1, 1, 1, 1}, {0, 1, 1, 1}, {0, 1, 1}, {0, 1}};
__constant__ uint8_t c_cdc_tz_len[3][4] = {{1, 2, 3, 3}, {1, 2, 2}, {1, 1}};
__constant__ uint8_t c_cdc_tz_bits[3][4] = {{1, 1, 1, 0}, {1, 1, 0}, {1, 0}};
// run_before (Table 9-10), [min(zerosLeft, 7) - 1][run_before]
__constant__ uint8_t c_run_len[7][15] = {{1, 1}, {1, 2, 2}, {2, 2, 2, 2}, {2, 2, 2, 3, 3}, {2, 2, 3, 3, 3, 3}, {2, 3, 3, 3, 3, 3, 3},
                                         {3, 3, 3, 3, 3, 3, 3, 4, 5, 6, 7, 8, 9, 10, 11}};
__constant__ uint8_t c_run_bits[7][15] = {{1, 0}, {1, 1, 0}, {3, 2, 1, 0}, {3, 2, 1, 1, 0}, {3, 2, 3, 2, 1, 0}, {3, 0, 1, 3, 2, 5, 4},
                                          {7, 6, 5, 4, 3, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1}};

struct Frame {
    int W, H, W16, H16, mbw, mbh;
    int qp;                    // the constant-QP stream's QP (kRc kernels read the picture's QP from rc)
    const uint8_t* rgb;
    uint8_t* cur;              // padded I420 of the input
    const uint8_t* ref;        // padded I420 reconstruction of the previous frame (P)
    uint8_t* rec;              // padded I420 reconstruction of this frame
    MbRec* mbs;
    int32_t* lens;             // bytes per slot, -1 when the slot overflowed
    int32_t* dbk;              // h264_deblock: [0] row ticket, [1 + r] MBs of row r filtered (reset on the stream per frame)
    int64_t* rc;               // rate-control state
    uint8_t* slots;
    int64_t slot_cap;
    int idr, frame_num, idr_pic_id;
    template <class T>         // component c (0 Y, 1 Cb, 2 Cr) of the padded I420 picture at base
    __device__ T* plane(T* base, int c) const { return base + (c == 0 ? 0 : (int64_t)W16 * H16 + (int64_t)(c - 1) * (W16 / 2) * (H16 / 2)); }
};

// The picture's QP: the constant one, or the controller's choice for this picture.
template <bool kRc>
__device__ __forceinline__ int pic_qp(const Frame& F) { return kRc ? (int)F.rc[kRcQp] : F.qp; }

// ------------------------------------------------------------------------------------------------ transforms and quantisation
__device__ __forceinline__ int cls4(int r) { const int i = r >> 2, j = r & 3; return ((i | j) & 1) == 0 ? 0 : ((i & j) & 1) ? 1 : 2; }

__device__ void fwd4(const int* x, int* w) {           // W = Cf X Cf^T, raster 4x4
    int t[16];
    for (int j = 0; j < 4; ++j) {                       // columns: Cf X
        const int a = x[j], b = x[4 + j], c = x[8 + j], d = x[12 + j];
        t[j] = a + b + c + d; t[4 + j] = 2 * a + b - c - 2 * d; t[8 + j] = a - b - c + d; t[12 + j] = a - 2 * b + 2 * c - d;
    }
    for (int i = 0; i < 4; ++i) {                       // rows: (Cf X) Cf^T
        const int a = t[4 * i], b = t[4 * i + 1], c = t[4 * i + 2], d = t[4 * i + 3];
        w[4 * i] = a + b + c + d; w[4 * i + 1] = 2 * a + b - c - 2 * d; w[4 * i + 2] = a - b - c + d; w[4 * i + 3] = a - 2 * b + 2 * c - d;
    }
}

__device__ void inv4(const int* d, int* r) {            // 8.5.12.2, then (x + 32) >> 6
    int f[16];
    for (int i = 0; i < 4; ++i) {
        const int* a = d + 4 * i;
        const int e0 = a[0] + a[2], e1 = a[0] - a[2], e2 = (a[1] >> 1) - a[3], e3 = a[1] + (a[3] >> 1);
        f[4 * i] = e0 + e3; f[4 * i + 1] = e1 + e2; f[4 * i + 2] = e1 - e2; f[4 * i + 3] = e0 - e3;
    }
    for (int j = 0; j < 4; ++j) {
        const int a0 = f[j], a1 = f[4 + j], a2 = f[8 + j], a3 = f[12 + j];
        const int e0 = a0 + a2, e1 = a0 - a2, e2 = (a1 >> 1) - a3, e3 = a1 + (a3 >> 1);
        r[j] = (e0 + e3 + 32) >> 6; r[4 + j] = (e1 + e2 + 32) >> 6; r[8 + j] = (e1 - e2 + 32) >> 6; r[12 + j] = (e0 - e3 + 32) >> 6;
    }
}

__device__ __forceinline__ int quant(int w, int mf, int qbits, int64_t f) {
    int l = (int)(((int64_t)abs(w) * mf + f) >> qbits);
    l = min(l, kLevelMax);
    return w < 0 ? -l : l;
}

__device__ __forceinline__ int64_t dz(int qp, bool intra) { return (int64_t)(1 << (15 + qp / 6)) / (intra ? 3 : 6); }

__device__ __forceinline__ int dequant(int c, int qp, int r) {
    const int ls = 16 * c_v[qp % 6][cls4(r)];
    return qp >= 24 ? (c * ls) * (1 << (qp / 6 - 4)) : (c * ls + (1 << (3 - qp / 6))) >> (4 - qp / 6);
}

// AC quantisation of one 4x4 block's coefficients w (raster) -> levels in zig-zag order (first = 0 skips the DC)
__device__ void quant_block(const int* w, int qp, bool intra, int first, int16_t* lv) {
    const int qbits = 15 + qp / 6;
    const int64_t f = dz(qp, intra);
    for (int k = 0; k < 16; ++k) {
        const int r = c_zz[k];
        lv[k] = k < first ? 0 : (int16_t)quant(w[r], c_mf[qp % 6][cls4(r)], qbits, f);
    }
}

// levels (zig-zag) -> residual samples (raster); dc >= INT_MIN + 1: already scaled DC (I_16x16 luma, chroma)
__device__ void recon_block(const int16_t* lv, int qp, bool has_dc, int dc, int* res) {
    int d[16];
    for (int k = 0; k < 16; ++k) d[c_zz[k]] = dequant(lv[k], qp, c_zz[k]);
    if (has_dc) d[0] = dc;
    inv4(d, res);
}

__device__ __forceinline__ int clip255(int v) { return min(max(v, 0), 255); }

__device__ __forceinline__ int ue_bits(unsigned k) { return 2 * (32 - __clz(k + 1)) - 1; }
__device__ __forceinline__ unsigned se_code(int v) { return v > 0 ? 2u * v - 1 : (unsigned)(-2 * v); }

// Chroma DC of one component: 2x2 transform of the four blocks' DC coefficients, quantise to lv[0..3], scale back to dcc[0..3]
__device__ void chroma_dc(const int* dc, int qpc, bool intra, int16_t* lv, int* dcc) {
    const int t[4] = {dc[0] + dc[1] + dc[2] + dc[3], dc[0] - dc[1] + dc[2] - dc[3], dc[0] + dc[1] - dc[2] - dc[3], dc[0] - dc[1] - dc[2] + dc[3]};
    const int mf = c_mf[qpc % 6][0], qbits = 16 + qpc / 6;
    const int64_t f = 2 * dz(qpc, intra);
    int c[4];
    for (int i = 0; i < 4; ++i) lv[i] = (int16_t)(c[i] = quant(t[i], mf, qbits, f));
    const int g[4] = {c[0] + c[1] + c[2] + c[3], c[0] - c[1] + c[2] - c[3], c[0] + c[1] - c[2] - c[3], c[0] - c[1] - c[2] + c[3]};
    const int ls = 16 * c_v[qpc % 6][0];
    for (int i = 0; i < 4; ++i) dcc[i] = (g[i] * ls * (1 << (qpc / 6))) >> 5;
}

// ------------------------------------------------------------------------------------------------ colour conversion
__global__ void h264_rgb_to_yuv(Frame F) {
    const int cw = F.W16 / 2, ch = F.H16 / 2;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < (int64_t)cw * ch; i += (int64_t)gridDim.x * blockDim.x) {
        const int cx = (int)(i % cw), cy = (int)(i / cw);
        uint8_t* Y = F.plane(F.cur, 0);
        for (int j = 0; j < 4; ++j) {
            const int x = 2 * cx + (j & 1), y = 2 * cy + (j >> 1);
            const uint8_t* p = F.rgb + ((int64_t)min(y, F.H - 1) * F.W + min(x, F.W - 1)) * 3;
            Y[(int64_t)y * F.W16 + x] = (uint8_t)(((66 * p[0] + 129 * p[1] + 25 * p[2] + 128) >> 8) + 16);
        }
        const int sx = min(cx, F.W / 2 - 1), sy = min(cy, F.H / 2 - 1);
        int sr = 0, sg = 0, sb = 0;
        for (int j = 0; j < 4; ++j) {
            const uint8_t* p = F.rgb + ((int64_t)(2 * sy + (j >> 1)) * F.W + 2 * sx + (j & 1)) * 3;
            sr += p[0]; sg += p[1]; sb += p[2];
        }
        F.plane(F.cur, 1)[(int64_t)cy * cw + cx] = (uint8_t)(((-38 * sr - 74 * sg + 112 * sb + 512) >> 10) + 128);
        F.plane(F.cur, 2)[(int64_t)cy * cw + cx] = (uint8_t)(((112 * sr - 94 * sg - 18 * sb + 512) >> 10) + 128);
    }
}

// ------------------------------------------------------------------------------------------------ IDR: I_16x16, one warp per row
template <bool kRc>
__global__ void __launch_bounds__(32) h264_intra_rows(Frame F) {
    __shared__ int s_w[16][16];        // luma coefficients per block (raster)
    __shared__ int s_cdc[2][4], s_dcc[2][4], s_dcy[16];
    __shared__ int s_left[16];
    const int row = blockIdx.x, lane = threadIdx.x;
    const int qp = pic_qp<kRc>(F), qpc = c_qpc[qp];
    const int cw = F.W16 / 2;
    const uint8_t* Ys = F.plane(F.cur, 0);
    uint8_t* Yr = F.plane(F.rec, 0);
    for (int mbx = 0; mbx < F.mbw; ++mbx) {
        MbRec* R = F.mbs + (int64_t)row * F.mbw + mbx;
        const int x0 = 16 * mbx, y0 = 16 * row;
        // luma mode: horizontal when its SAD is not larger than DC's (lower mode number wins ties); DC only without a left MB
        if (lane < 16) s_left[lane] = mbx ? Yr[(int64_t)(y0 + lane) * F.W16 + x0 - 1] : 128;
        __syncwarp();
        int sum = 0;
        for (int i = 0; i < 16; ++i) sum += s_left[i];
        const int dcp = mbx ? (sum + 8) >> 4 : 128;
        int sad_h = 0, sad_dc = 0;
        if (lane < 16) {
            for (int x = 0; x < 16; ++x) {
                const int s = Ys[(int64_t)(y0 + lane) * F.W16 + x0 + x];
                sad_h += abs(s - s_left[lane]);
                sad_dc += abs(s - dcp);
            }
        }
        for (int o = 16; o; o >>= 1) {
            sad_h += __shfl_xor_sync(0xffffffffu, sad_h, o);
            sad_dc += __shfl_xor_sync(0xffffffffu, sad_dc, o);
        }
        const int mode = (mbx && sad_h <= sad_dc) ? 1 : 2;
        // forward transforms: lanes 0-15 luma blocks, 16-23 chroma blocks
        int w[16], res[16];
        const int bx = lane < 16 ? c_blk_x[lane] : ((lane - 16) & 1), by = lane < 16 ? c_blk_y[lane] : (((lane - 16) >> 1) & 1);
        const int comp = lane < 16 ? 0 : 1 + ((lane - 16) >> 2);
        int pred[16];
        if (lane < 16) {
            for (int r = 0; r < 16; ++r) {
                const int y = 4 * by + (r >> 2), x = 4 * bx + (r & 3);
                pred[r] = mode == 1 ? s_left[y] : dcp;
                w[r] = Ys[(int64_t)(y0 + y) * F.W16 + x0 + x] - pred[r];
            }
            fwd4(w, s_w[lane]);
        } else if (lane < 24) {
            const uint8_t* Cs = F.plane(F.cur, comp);
            const uint8_t* Cr = F.plane(F.rec, comp);
            int p = 128;
            if (mbx) {
                int s = 0;
                for (int i = 0; i < 4; ++i) s += Cr[(int64_t)(8 * row + 4 * by + i) * cw + 8 * mbx - 1];
                p = (s + 2) >> 2;
            }
            for (int r = 0; r < 16; ++r) {
                pred[r] = p;
                w[r] = Cs[(int64_t)(8 * row + 4 * by + (r >> 2)) * cw + 8 * mbx + 4 * bx + (r & 3)] - p;
            }
            fwd4(w, w);
            s_cdc[comp - 1][(lane - 16) & 3] = w[0];
        }
        __syncwarp();
        if (lane == 0) {                                 // luma DC: Hadamard, quantise, inverse, scale
            int m[16], t[16], c[16];
            for (int k = 0; k < 16; ++k) m[4 * c_blk_y[k] + c_blk_x[k]] = s_w[k][0];
            for (int j = 0; j < 4; ++j) {
                const int a = m[j], b = m[4 + j], cc = m[8 + j], d = m[12 + j];
                t[j] = a + b + cc + d; t[4 + j] = a + b - cc - d; t[8 + j] = a - b - cc + d; t[12 + j] = a - b + cc - d;
            }
            for (int i = 0; i < 4; ++i) {
                const int a = t[4 * i], b = t[4 * i + 1], cc = t[4 * i + 2], d = t[4 * i + 3];
                m[4 * i] = (a + b + cc + d) >> 1; m[4 * i + 1] = (a + b - cc - d) >> 1; m[4 * i + 2] = (a - b - cc + d) >> 1; m[4 * i + 3] = (a - b + cc - d) >> 1;
            }
            const int mf = c_mf[qp % 6][0], qbits = 16 + qp / 6;
            const int64_t f = 2 * dz(qp, true);
            for (int r = 0; r < 16; ++r) c[r] = quant(m[r], mf, qbits, f);
            for (int k = 0; k < 16; ++k) R->lv[16][k] = (int16_t)c[c_zz[k]];
            for (int j = 0; j < 4; ++j) {
                const int a = c[j], b = c[4 + j], cc = c[8 + j], d = c[12 + j];
                t[j] = a + b + cc + d; t[4 + j] = a + b - cc - d; t[8 + j] = a - b - cc + d; t[12 + j] = a - b + cc - d;
            }
            const int ls = 16 * c_v[qp % 6][0];
            for (int i = 0; i < 4; ++i) {
                const int a = t[4 * i], b = t[4 * i + 1], cc = t[4 * i + 2], d = t[4 * i + 3];
                const int g[4] = {a + b + cc + d, a + b - cc - d, a - b - cc + d, a - b + cc - d};
                for (int j = 0; j < 4; ++j)
                    m[4 * i + j] = qp >= 36 ? (g[j] * ls) * (1 << (qp / 6 - 6)) : (g[j] * ls + (1 << (5 - qp / 6))) >> (6 - qp / 6);
            }
            for (int k = 0; k < 16; ++k) s_dcy[k] = m[4 * c_blk_y[k] + c_blk_x[k]];
            R->mode = mode;
            R->mvx = R->mvy = 0;
        } else if (lane == 1 || lane == 2) {
            chroma_dc(s_cdc[lane - 1], qpc, true, R->lv[17] + 4 * (lane - 1), s_dcc[lane - 1]);
            for (int k = 0; k < 4; ++k) R->lv[17][8 + 4 * (lane - 1) + k] = 0;
        }
        __syncwarp();
        if (lane < 16) {
            quant_block(s_w[lane], qp, true, 1, R->lv[lane]);
            recon_block(R->lv[lane], qp, true, s_dcy[lane], res);
            for (int r = 0; r < 16; ++r)
                Yr[(int64_t)(y0 + 4 * by + (r >> 2)) * F.W16 + x0 + 4 * bx + (r & 3)] = (uint8_t)clip255(pred[r] + res[r]);
        } else if (lane < 24) {
            int16_t* lv = R->lv[18 + (lane - 16)];
            quant_block(w, qpc, true, 1, lv);
            recon_block(lv, qpc, true, s_dcc[comp - 1][(lane - 16) & 3], res);
            uint8_t* Cr = F.plane(F.rec, comp);
            for (int r = 0; r < 16; ++r)
                Cr[(int64_t)(8 * row + 4 * by + (r >> 2)) * cw + 8 * mbx + 4 * bx + (r & 3)] = (uint8_t)clip255(pred[r] + res[r]);
        }
        __syncwarp();
    }
}

// Luma sample at quarter-sample position (X4, Y4) of patch p (8.4.2.2.1, Table 8-12): the 6-tap half samples b (right), h (below)
// and j (both), the quarter samples averages of their neighbours.  The position must keep 2 samples left / above and 3 right / below.
__device__ int qpel(const uint8_t (*p)[kPat], int X4, int Y4) {
    const int x = X4 >> 2, y = Y4 >> 2;
    auto G = [&](int yy, int xx) { return (int)p[yy][xx]; };
    auto b1 = [&](int yy, int xx) { return G(yy, xx - 2) - 5 * G(yy, xx - 1) + 20 * G(yy, xx) + 20 * G(yy, xx + 1) - 5 * G(yy, xx + 2) + G(yy, xx + 3); };
    auto B = [&](int yy, int xx) { return clip255((b1(yy, xx) + 16) >> 5); };
    auto Hh = [&](int yy, int xx) {
        return clip255((G(yy - 2, xx) - 5 * G(yy - 1, xx) + 20 * G(yy, xx) + 20 * G(yy + 1, xx) - 5 * G(yy + 2, xx) + G(yy + 3, xx) + 16) >> 5);
    };
    auto J = [&]() {
        return clip255((b1(y - 2, x) - 5 * b1(y - 1, x) + 20 * b1(y, x) + 20 * b1(y + 1, x) - 5 * b1(y + 2, x) + b1(y + 3, x) + 512) >> 10);
    };
    auto av = [](int a, int c) { return (a + c + 1) >> 1; };
    switch (4 * (Y4 & 3) + (X4 & 3)) {
        case 0: return G(y, x);
        case 1: return av(G(y, x), B(y, x));
        case 2: return B(y, x);
        case 3: return av(G(y, x + 1), B(y, x));
        case 4: return av(G(y, x), Hh(y, x));
        case 5: return av(B(y, x), Hh(y, x));
        case 6: return av(B(y, x), J());
        case 7: return av(B(y, x), Hh(y, x + 1));
        case 8: return Hh(y, x);
        case 9: return av(Hh(y, x), J());
        case 10: return J();
        case 11: return av(J(), Hh(y, x + 1));
        case 12: return av(G(y + 1, x), Hh(y, x));
        case 13: return av(Hh(y, x), B(y + 1, x));
        case 14: return av(J(), B(y + 1, x));
        default: return av(Hh(y, x + 1), B(y + 1, x));
    }
}

__device__ __forceinline__ unsigned long long mv_key(int cost, int qx, int qy) {
    return ((unsigned long long)cost << 24) | ((unsigned long long)(abs(qx) + abs(qy)) << 16) | ((unsigned long long)(qy + kMvOff) << 8) |
           (unsigned long long)(qx + kMvOff);
}

// ------------------------------------------------------------------------------------------------ P: one block per MB
template <bool kRc>
__global__ void __launch_bounds__(256) h264_inter_mbs(Frame F) {
    __shared__ uint8_t s_win[kWin][kWin];
    __shared__ uint8_t s_cur[16][16];
    __shared__ unsigned long long s_best[8];
    __shared__ int s_cdc[2][4], s_dcc[2][4];
    const int mbx = blockIdx.x, row = blockIdx.y, tid = threadIdx.x;
    const int qp = pic_qp<kRc>(F), qpc = c_qpc[qp];
    const int x0 = 16 * mbx, y0 = 16 * row;
    const uint8_t* Yref = F.plane(F.ref, 0);
    const uint8_t* Ys = F.plane(F.cur, 0);
    for (int i = tid; i < kWin * kWin; i += 256) {
        const int y = min(max(y0 - kSearch + i / kWin, 0), F.H16 - 1), x = min(max(x0 - kSearch + i % kWin, 0), F.W16 - 1);
        s_win[i / kWin][i % kWin] = Yref[(int64_t)y * F.W16 + x];
    }
    s_cur[tid >> 4][tid & 15] = Ys[(int64_t)(y0 + (tid >> 4)) * F.W16 + x0 + (tid & 15)];
    __syncthreads();
    // cost = SAD + lambda * bits of the MV against a zero predictor (so that MBs are decided independently); ties: smaller
    // |mvx| + |mvy|, then smaller (mvy, mvx)
    const int lam = c_lambda[qp];
    unsigned long long best = ~0ull;
    for (int c = tid; c < kCands; c += 256) {
        const int my = c / (2 * kSearch + 1) - kSearch, mx = c % (2 * kSearch + 1) - kSearch;
        int sad = 0;
        for (int y = 0; y < 16; ++y) {
            const uint8_t* wr = &s_win[kSearch + my + y][kSearch + mx];
#pragma unroll
            for (int x = 0; x < 16; ++x) sad += abs((int)s_cur[y][x] - (int)wr[x]);
        }
        best = min(best, mv_key(sad + lam * (ue_bits(se_code(4 * mx)) + ue_bits(se_code(4 * my))), 4 * mx, 4 * my));
    }
    for (int o = 16; o; o >>= 1) best = min(best, __shfl_xor_sync(0xffffffffu, best, o));
    if ((tid & 31) == 0) s_best[tid >> 5] = best;
    __syncthreads();
    best = s_best[0];
    for (int i = 1; i < 8; ++i) best = min(best, s_best[i]);
    int qx = (int)(best & 0xff) - kMvOff, qy = (int)((best >> 8) & 0xff) - kMvOff;
    const int mvx = qx / 4, mvy = qy / 4;                // the integer-pel vector
    // quarter-sample refinement (rate-controlled stream): the 8 half-sample neighbours of the integer vector, then the 8
    // quarter-sample neighbours of the best of those, same cost and tie order; one warp per candidate over a haloed patch
    __shared__ uint8_t s_pat[kRc ? kPat : 1][kPat];
    __shared__ unsigned long long s_key[8];
    if constexpr (kRc) {
        for (int i = tid; i < kPat * kPat; i += 256) {
            const int y = min(max(y0 + mvy - 3 + i / kPat, 0), F.H16 - 1), x = min(max(x0 + mvx - 3 + i % kPat, 0), F.W16 - 1);
            s_pat[i / kPat][i % kPat] = Yref[(int64_t)y * F.W16 + x];
        }
        __syncthreads();
        const int warp = tid >> 5, lane32 = tid & 31;
        for (int step = 2; step >= 1; --step) {
            const int cx = qx, cy = qy;
            const int d = warp < 4 ? warp : warp + 1, dx = d % 3 - 1, dy = d / 3 - 1;
            const int x4 = cx + step * dx, y4 = cy + step * dy;
            int sad = 0;
            for (int k = 0; k < 8; ++k) {
                const int pix = lane32 + 32 * k, y = pix >> 4, x = pix & 15;
                sad += abs((int)s_cur[y][x] - qpel(s_pat, 4 * (x + 3) + x4 - 4 * mvx, 4 * (y + 3) + y4 - 4 * mvy));
            }
            for (int o = 16; o; o >>= 1) sad += __shfl_xor_sync(0xffffffffu, sad, o);
            if (lane32 == 0) s_key[warp] = mv_key(sad + lam * (ue_bits(se_code(x4)) + ue_bits(se_code(y4))), x4, y4);
            __syncthreads();
            for (int i = 0; i < 8; ++i) best = min(best, s_key[i]);
            __syncthreads();
            qx = (int)(best & 0xff) - kMvOff;
            qy = (int)((best >> 8) & 0xff) - kMvOff;
        }
    }
    MbRec* R = F.mbs + (int64_t)row * F.mbw + mbx;
    const int cw = F.W16 / 2, chh = F.H16 / 2;
    int w[16], pred[16], res[16];
    const int lane = tid;
    const int bx = lane < 16 ? c_blk_x[lane] : ((lane - 16) & 1), by = lane < 16 ? c_blk_y[lane] : (((lane - 16) >> 1) & 1);
    const int comp = lane < 16 ? 0 : 1 + ((lane - 16) >> 2);
    if (lane < 16) {
        for (int r = 0; r < 16; ++r) {
            const int y = 4 * by + (r >> 2), x = 4 * bx + (r & 3);
            pred[r] = kRc ? qpel(s_pat, 4 * (x + 3) + qx - 4 * mvx, 4 * (y + 3) + qy - 4 * mvy) : s_win[kSearch + mvy + y][kSearch + mvx + x];
            w[r] = s_cur[y][x] - pred[r];
        }
        fwd4(w, w);
        quant_block(w, qp, false, 0, R->lv[lane]);
        recon_block(R->lv[lane], qp, false, 0, res);
        uint8_t* Yr = F.plane(F.rec, 0);
        for (int r = 0; r < 16; ++r)
            Yr[(int64_t)(y0 + 4 * by + (r >> 2)) * F.W16 + x0 + 4 * bx + (r & 3)] = (uint8_t)clip255(pred[r] + res[r]);
    } else if (lane < 24) {                              // chroma: eighth-pel bilinear at the luma MV (8.4.2.2.2)
        const int mvcx = qx, mvcy = qy, fx = mvcx & 7, fy = mvcy & 7;      // chroma eighth samples = luma quarter samples
        const uint8_t* Cref = F.plane(F.ref, comp);
        const uint8_t* Cs = F.plane(F.cur, comp);
        for (int r = 0; r < 16; ++r) {
            const int yy = 8 * row + 4 * by + (r >> 2), xx = 8 * mbx + 4 * bx + (r & 3);
            const int ry = yy + (mvcy >> 3), rx = xx + (mvcx >> 3);
            auto at = [&](int y, int x) { return (int)Cref[(int64_t)min(max(y, 0), chh - 1) * cw + min(max(x, 0), cw - 1)]; };
            pred[r] = ((8 - fx) * (8 - fy) * at(ry, rx) + fx * (8 - fy) * at(ry, rx + 1) + (8 - fx) * fy * at(ry + 1, rx) + fx * fy * at(ry + 1, rx + 1) + 32) >> 6;
            w[r] = Cs[(int64_t)yy * cw + xx] - pred[r];
        }
        fwd4(w, w);
        s_cdc[comp - 1][(lane - 16) & 3] = w[0];
    } else if (lane == 32) {
        R->mode = 0;
        R->mvx = qx;
        R->mvy = qy;
        for (int k = 0; k < 16; ++k) R->lv[16][k] = 0;
    }
    __syncthreads();
    if (lane == 0 || lane == 1) {
        chroma_dc(s_cdc[lane], qpc, false, R->lv[17] + 4 * lane, s_dcc[lane]);
        for (int k = 0; k < 4; ++k) R->lv[17][8 + 4 * lane + k] = 0;
    }
    __syncthreads();
    if (lane >= 16 && lane < 24) {
        int16_t* lv = R->lv[18 + (lane - 16)];
        quant_block(w, qpc, false, 1, lv);
        recon_block(lv, qpc, true, s_dcc[comp - 1][(lane - 16) & 3], res);
        uint8_t* Cr = F.plane(F.rec, comp);
        for (int r = 0; r < 16; ++r)
            Cr[(int64_t)(8 * row + 4 * by + (r >> 2)) * cw + 8 * mbx + 4 * bx + (r & 3)] = (uint8_t)clip255(pred[r] + res[r]);
    }
}

// ------------------------------------------------------------------------------------------------ deblocking (8.7)
// One edge line: q points at q0, step = distance from q0 to q1 (p_k = q[-(k + 1) * step], q_k = q[k * step]).  Loads bypass L1
// (other CTAs write the rows above during the kernel).
__device__ void filter_line(uint8_t* q, int64_t step, int bS, int idx, bool chroma) {
    if (bS == 0) return;
    const int a = c_alpha[idx], be = c_beta[idx];
    auto ld = [&](int k) { return (int)__ldcg(q + k * step); };
    const int p0 = ld(-1), q0 = ld(0), p1 = ld(-2), q1 = ld(1);
    if (abs(p0 - q0) >= a || abs(p1 - p0) >= be || abs(q1 - q0) >= be) return;
    if (chroma) {
        if (bS < 4) {
            const int tc = c_tc0[idx][bS - 1] + 1;
            const int delta = min(max((((q0 - p0) << 2) + (p1 - q1) + 4) >> 3, -tc), tc);
            q[-step] = (uint8_t)clip255(p0 + delta);
            q[0] = (uint8_t)clip255(q0 - delta);
        } else {
            q[-step] = (uint8_t)((2 * p1 + p0 + q1 + 2) >> 2);
            q[0] = (uint8_t)((2 * q1 + q0 + p1 + 2) >> 2);
        }
        return;
    }
    const int p2 = ld(-3), q2 = ld(2);
    const bool ap = abs(p2 - p0) < be, aq = abs(q2 - q0) < be;
    if (bS < 4) {
        const int tc0 = c_tc0[idx][bS - 1], tc = tc0 + ap + aq;
        const int delta = min(max((((q0 - p0) << 2) + (p1 - q1) + 4) >> 3, -tc), tc);
        q[-step] = (uint8_t)clip255(p0 + delta);
        q[0] = (uint8_t)clip255(q0 - delta);
        if (ap) q[-2 * step] = (uint8_t)(p1 + min(max((p2 + ((p0 + q0 + 1) >> 1) - (p1 << 1)) >> 1, -tc0), tc0));
        if (aq) q[step] = (uint8_t)(q1 + min(max((q2 + ((p0 + q0 + 1) >> 1) - (q1 << 1)) >> 1, -tc0), tc0));
        return;
    }
    const bool near = abs(p0 - q0) < ((a >> 2) + 2);
    if (ap && near) {
        const int p3 = ld(-4);
        q[-step] = (uint8_t)((p2 + 2 * p1 + 2 * p0 + 2 * q0 + q1 + 4) >> 3);
        q[-2 * step] = (uint8_t)((p2 + p1 + p0 + q0 + 2) >> 2);
        q[-3 * step] = (uint8_t)((2 * p3 + 3 * p2 + p1 + p0 + q0 + 4) >> 3);
    } else {
        q[-step] = (uint8_t)((2 * p1 + p0 + q1 + 2) >> 2);
    }
    if (aq && near) {
        const int q3 = ld(3);
        q[0] = (uint8_t)((p1 + 2 * p0 + 2 * q0 + 2 * q1 + q2 + 4) >> 3);
        q[step] = (uint8_t)((p0 + q0 + q1 + q2 + 2) >> 2);
        q[2 * step] = (uint8_t)((2 * q3 + 3 * q2 + q1 + q0 + p0 + 4) >> 3);
    } else {
        q[0] = (uint8_t)((2 * q1 + q0 + p1 + 2) >> 2);
    }
}

// Bit (4 * by + bx) set when luma 4x4 block (bx, by) of the MB has nonzero levels; lanes 0-15 of a warp.
__device__ unsigned nz_mask(const MbRec* R, int lane) {
    bool nz = false;
    for (int i = 0; lane < 16 && i < 16; ++i) nz |= R->lv[lane][i] != 0;
    const unsigned b = __ballot_sync(0xffffffffu, nz);
    unsigned m = 0;
    for (int k = 0; k < 16; ++k) if (b >> k & 1) m |= 1u << (4 * c_blk_y[k] + c_blk_x[k]);
    return m;
}

// bS (8.7.2.1) of the luma edge between 4x4 blocks p and q: intra picture 4 on MB edges, 3 inside; else 2 when either block has
// levels, 1 on MB edges whose vectors differ by >= 4 quarter samples in a component, 0 otherwise.
__device__ __forceinline__ int bs_of(bool intra, bool mb_edge, bool nz, bool mv_differs) {
    if (intra) return mb_edge ? 4 : 3;
    return nz ? 2 : (mb_edge && mv_differs) ? 1 : 0;
}

// One warp per MB row, rows in ticket order; lanes 0-15 own a luma line of the edge being filtered, lanes 16-23 a Cb line, 24-31 a
// Cr line.  Per MB: vertical edges left to right, then horizontal edges top to bottom.  MB x of row r starts once row r - 1 has
// finished MB x + 1, the last MB whose filtering touches the samples MB x reads.
__global__ void __launch_bounds__(32) h264_deblock(Frame F) {
    __shared__ int s_row;
    const int lane = threadIdx.x;
    if (lane == 0) s_row = atomicAdd(F.dbk, 1);
    __syncwarp();
    const int row = s_row;
    const int qp = pic_qp<true>(F), qpc = c_qpc[qp];
    const bool intra = F.idr;
    volatile int32_t* done = F.dbk + 1;
    const int cw = F.W16 / 2;
    uint8_t* Y = F.plane(F.rec, 0);
    uint8_t* Cp = F.plane(F.rec, lane < 24 ? 1 : 2);
    const int line = lane < 16 ? lane : (lane - 16) & 7;
    unsigned nz_left = 0;
    for (int mbx = 0; mbx < F.mbw; ++mbx) {
        if (row > 0 && lane == 0) {
            const int need = min(mbx + 2, F.mbw);
            uint32_t it = 0;
            while (done[row - 1] < need) {
                if (++it == kSpinLimit) __trap();
                __nanosleep(64);
            }
            __threadfence();
        }
        __syncwarp();
        const MbRec* R = F.mbs + (int64_t)row * F.mbw + mbx;
        const unsigned nz = intra ? 0u : nz_mask(R, lane);
        const unsigned nz_top = (intra || row == 0) ? 0u : nz_mask(R - F.mbw, lane);
        const int x0 = 16 * mbx, y0 = 16 * row;
        for (int dir = 0; dir < 2; ++dir) {                  // 0: vertical edges, 1: horizontal edges
            const bool has_prev = dir ? row > 0 : mbx > 0;
            const unsigned nz_prev = dir ? nz_top : nz_left;
            const MbRec* P = dir ? R - F.mbw : R - 1;
            const bool mvd = has_prev && !intra && (abs(R->mvx - P->mvx) >= 4 || abs(R->mvy - P->mvy) >= 4);
            for (int e = 0; e < 4; ++e) {
                if (e == 0 && !has_prev) continue;
                const int blk = (lane < 16 ? line : 2 * line) >> 2;    // 4x4 block index along the edge
                // nz of the blocks either side: bit (4 * by + bx); vertical edges: bx = e - 1 | e, by = blk
                const int qb = dir ? 4 * e + blk : 4 * blk + e;
                const bool nzq = nz >> qb & 1;
                const bool nzp = e ? (nz >> (dir ? qb - 4 : qb - 1) & 1) : (nz_prev >> (dir ? 12 + blk : 4 * blk + 3) & 1);
                const int bS = bs_of(intra, e == 0, nzp || nzq, mvd);
                if (lane < 16) {
                    uint8_t* q = dir ? Y + (int64_t)(y0 + 4 * e) * F.W16 + x0 + line : Y + (int64_t)(y0 + line) * F.W16 + x0 + 4 * e;
                    filter_line(q, dir ? F.W16 : 1, bS, qp, false);
                } else if (!(e & 1)) {
                    uint8_t* q = dir ? Cp + (int64_t)(8 * row + 2 * e) * cw + 8 * mbx + line : Cp + (int64_t)(8 * row + line) * cw + 8 * mbx + 2 * e;
                    filter_line(q, dir ? cw : 1, bS, qpc, true);
                }
                __syncwarp();
            }
        }
        nz_left = nz;
        __threadfence();
        __syncwarp();
        if (lane == 0) done[row] = mbx + 1;
    }
}

// ------------------------------------------------------------------------------------------------ rate control
__device__ __forceinline__ int64_t floor_div(int64_t a, int64_t b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }

// First QP from bits per pixel: 30 at 0.1, 6 less per doubling, clamped to the bounds.
__global__ void h264_rc_init(int64_t* st, int width, int height, int64_t bitrate, int64_t num, int64_t den, int qp_min, int qp_max) {
    for (int i = 0; i < kRcFields; ++i) st[i] = 0;
    st[kRcBitrate] = bitrate; st[kRcNum] = num; st[kRcDen] = den; st[kRcQpMin] = qp_min; st[kRcQpMax] = qp_max;
    int64_t x = 10 * bitrate * den, y = num * width * height;
    int q = 30;
    while (x >= 2 * y && q > 0) { y *= 2; q -= 6; }
    while (2 * x < y && q < 51) { x *= 2; q += 6; }
    st[kRcQp] = min(max(q, qp_min), qp_max);
}

// After a frame: fullness += its bits - bitrate / fps (saturating at +-8 s); after a P frame, or an IDR frame that follows an IDR
// frame, QP moves by -2..+2 by the ratio of the frame's bits to its budget (the per-frame rate less a second's share of the
// fullness, at least 1/8 of the rate).  IDR frames keep the QP of the P frames around them.
__global__ void h264_rc_update(int64_t* st, const int64_t* sample_len, int idr) {
    const int64_t len = *sample_len;
    if (len < 0) return;                                 // overflowed slot: the writer reports it
    const int64_t num = st[kRcNum], budget = st[kRcBitrate] * st[kRcDen], sat = 8 * st[kRcBitrate] * num;
    const int64_t bits = 8 * len * num;
    const int64_t full = min(max(st[kRcFullness] + bits - budget, -sat), sat);
    st[kRcFullness] = full;
    if (!idr || st[kRcPrevIdr]) {
        const int64_t want = max(budget - floor_div(full, max(num / st[kRcDen], (int64_t)1)), budget / 8);
        const int step = 100 * bits > 141 * want ? 2 : 100 * bits > 112 * want ? 1 : 141 * bits < 100 * want ? -2 : 112 * bits < 100 * want ? -1 : 0;
        st[kRcQp] = min(max(st[kRcQp] + step, st[kRcQpMin]), st[kRcQpMax]);
    }
    st[kRcPrevIdr] = idr;
    st[kRcFrames] += 1;
}

// ------------------------------------------------------------------------------------------------ CAVLC slice writer
struct BitWriter {
    uint8_t* out;
    int64_t cap, pos;
    uint64_t acc;
    int n, zeros;
    bool overflow;
    __device__ void emit(uint8_t b) {
        if (pos < cap) out[pos] = b; else overflow = true;
        ++pos;
    }
    __device__ void byte(uint8_t b) {                  // emulation prevention: 0x000003 before 0x000000 .. 0x000003
        if (zeros >= 2 && b <= 3) { emit(3); zeros = 0; }
        emit(b);
        zeros = b ? 0 : zeros + 1;
    }
    __device__ void u(uint32_t v, int nb) {            // nb <= 32
        if (!nb) return;
        acc = (acc << nb) | (v & (uint32_t)((1ull << nb) - 1));
        n += nb;
        while (n >= 8) { n -= 8; byte((uint8_t)(acc >> n)); }
    }
    __device__ void ue(uint32_t k) {
        const int len = 32 - __clz(k + 1);
        u(0, len - 1);
        u(k + 1, len);
    }
    __device__ void se(int v) { ue(se_code(v)); }
    __device__ void trailing() { u(1, 1); if (n) u(0, 8 - n); }
};

__device__ __forceinline__ int nc_of(int na, int nb) {          // -1: not available
    if (na >= 0 && nb >= 0) return (na + nb + 1) >> 1;
    return na >= 0 ? na : nb >= 0 ? nb : 0;
}

// residual_block_cavlc (9.2) of n levels (zig-zag order); nc = -1: chroma DC.  Returns TotalCoeff.
__device__ int residual_block(BitWriter& bw, const int16_t* c, int n, int nc) {
    int pos[16], total = 0;
    for (int i = 0; i < n; ++i) if (c[i]) pos[total++] = i;
    int t1 = 0;
    for (int k = total - 1; k >= 0 && t1 < 3 && abs(c[pos[k]]) == 1; --k) ++t1;
    const int idx = 4 * total + t1;
    if (nc == -1) {
        bw.u(c_cdc_ct_bits[idx], c_cdc_ct_len[idx]);
    } else {
        const int tab = nc < 2 ? 0 : nc < 4 ? 1 : nc < 8 ? 2 : 3;
        bw.u(c_ct_bits[tab][idx], c_ct_len[tab][idx]);
    }
    if (!total) return 0;
    for (int k = 0; k < t1; ++k) bw.u(c[pos[total - 1 - k]] < 0, 1);
    int sl = (total > 10 && t1 < 3) ? 1 : 0;
    for (int k = t1; k < total; ++k) {
        const int lv = c[pos[total - 1 - k]];
        int code = lv > 0 ? 2 * lv - 2 : -2 * lv - 1;
        if (k == t1 && t1 < 3) code -= 2;
        int prefix, sbits, sval;
        if (sl == 0) {
            if (code < 14) { prefix = code; sbits = 0; sval = 0; }
            else if (code < 30) { prefix = 14; sbits = 4; sval = code - 14; }
            else { prefix = 15; sbits = 12; sval = code - 30; }
        } else if (code < (15 << sl)) {
            prefix = code >> sl; sbits = sl; sval = code & ((1 << sl) - 1);
        } else {
            prefix = 15; sbits = 12; sval = code - (15 << sl);
        }
        bw.u(1, prefix + 1);
        bw.u(sval, sbits);
        if (sl == 0) sl = 1;
        if (abs(lv) > (3 << (sl - 1)) && sl < 6) ++sl;
    }
    if (total < n) {
        const int tz = pos[total - 1] + 1 - total;
        if (nc == -1) bw.u(c_cdc_tz_bits[total - 1][tz], c_cdc_tz_len[total - 1][tz]);
        else bw.u(c_tz_bits[total - 1][tz], c_tz_len[total - 1][tz]);
        int left = tz;
        for (int j = total - 1; j > 0 && left > 0; --j) {
            const int run = pos[j] - pos[j - 1] - 1, t = min(left, 7) - 1;
            bw.u(c_run_bits[t][run], c_run_len[t][run]);
            left -= run;
        }
    }
    return total;
}

__device__ bool any_nonzero(const int16_t* p, int n) {
    for (int i = 0; i < n; ++i) if (p[i]) return true;
    return false;
}

template <bool kRc>
__global__ void h264_write_rows(Frame F) {
    const int row = blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= F.mbh) return;
    uint8_t* slot = F.slots + row * F.slot_cap;
    BitWriter bw{slot + 5, F.slot_cap - 5, 0, 0, 0, 0, false};
    const bool idr = F.idr;
    bw.ue(row * F.mbw);                      // first_mb_in_slice
    bw.ue(idr ? 2 : 0);                      // slice_type I / P
    bw.ue(0);                                // pic_parameter_set_id
    bw.u(F.frame_num, 4);                    // frame_num (log2_max_frame_num = 4)
    if (idr) {
        bw.ue(F.idr_pic_id);
    } else {
        bw.u(0, 1);                          // num_ref_idx_active_override_flag
        bw.u(0, 1);                          // ref_pic_list_modification_flag_l0
    }
    bw.u(0, 1);                              // no_output_of_prior_pics_flag / adaptive_ref_pic_marking_mode_flag
    if (idr) bw.u(0, 1);                     // long_term_reference_flag
    if (kRc) {
        bw.se(pic_qp<kRc>(F) - 26);          // slice_qp_delta (pic_init_qp 26)
        bw.ue(0);                            // disable_deblocking_filter_idc: filter, across slice boundaries too
        bw.se(0);                            // slice_alpha_c0_offset_div2
        bw.se(0);                            // slice_beta_offset_div2
    } else {
        bw.se(0);                            // slice_qp_delta
        bw.ue(1);                            // disable_deblocking_filter_idc
    }
    int left_tc[4] = {0, 0, 0, 0}, left_cc[2][2] = {{0, 0}, {0, 0}};
    int skip_run = 0, mvpx = 0, mvpy = 0;
    for (int mbx = 0; mbx < F.mbw; ++mbx) {
        const MbRec* R = F.mbs + (int64_t)row * F.mbw + mbx;
        const bool left = mbx > 0;
        if (!idr && R->mvx == 0 && R->mvy == 0 && !any_nonzero(&R->lv[0][0], 26 * 16)) {     // P_Skip
            ++skip_run;
            for (int i = 0; i < 4; ++i) left_tc[i] = 0;
            left_cc[0][0] = left_cc[0][1] = left_cc[1][0] = left_cc[1][1] = 0;
            mvpx = mvpy = 0;
            continue;
        }
        int cbp_l = 0;
        if (idr) {
            for (int k = 0; k < 16 && !cbp_l; ++k) if (any_nonzero(R->lv[k] + 1, 15)) cbp_l = 15;
        } else {
            for (int k = 0; k < 16; ++k) if (any_nonzero(R->lv[k], 16)) cbp_l |= 1 << (k >> 2);
        }
        bool cac = false;
        for (int k = 0; k < 8 && !cac; ++k) cac = any_nonzero(R->lv[18 + k] + 1, 15);
        const int cbp_c = cac ? 2 : any_nonzero(R->lv[17], 8) ? 1 : 0;
        if (idr) {
            bw.ue(1 + R->mode + 4 * cbp_c + (cbp_l ? 12 : 0));     // mb_type I_16x16
            bw.ue(0);                                            // intra_chroma_pred_mode DC
            bw.se(0);                                            // mb_qp_delta
            residual_block(bw, R->lv[16], 16, left ? left_tc[0] : 0);
        } else {
            bw.ue(skip_run);
            skip_run = 0;
            bw.ue(0);                                            // mb_type P_L0_16x16
            bw.se(R->mvx - mvpx);
            bw.se(R->mvy - mvpy);
            mvpx = R->mvx;
            mvpy = R->mvy;
            bw.ue(c_inter_cbp_code[cbp_l + 16 * cbp_c]);
            if (cbp_l || cbp_c) bw.se(0);                        // mb_qp_delta
        }
        int tc[4][4] = {};
        for (int k = 0; k < 16; ++k) {
            if (!(cbp_l >> (k >> 2) & 1)) continue;
            const int bx = c_blk_x[k], by = c_blk_y[k];
            const int na = bx ? tc[by][bx - 1] : left ? left_tc[by] : -1, nb = by ? tc[by - 1][bx] : -1;
            tc[by][bx] = idr ? residual_block(bw, R->lv[k] + 1, 15, nc_of(na, nb)) : residual_block(bw, R->lv[k], 16, nc_of(na, nb));
        }
        int cc[2][2][2] = {};
        if (cbp_c) {
            residual_block(bw, R->lv[17], 4, -1);
            residual_block(bw, R->lv[17] + 4, 4, -1);
        }
        if (cbp_c == 2) {
            for (int comp = 0; comp < 2; ++comp)
                for (int k = 0; k < 4; ++k) {
                    const int bx = k & 1, by = k >> 1;
                    const int na = bx ? cc[comp][by][0] : left ? left_cc[comp][by] : -1, nb = by ? cc[comp][0][bx] : -1;
                    cc[comp][by][bx] = residual_block(bw, R->lv[18 + 4 * comp + k] + 1, 15, nc_of(na, nb));
                }
        }
        for (int i = 0; i < 4; ++i) left_tc[i] = tc[i][3];
        for (int comp = 0; comp < 2; ++comp) { left_cc[comp][0] = cc[comp][0][1]; left_cc[comp][1] = cc[comp][1][1]; }
    }
    if (skip_run) bw.ue(skip_run);
    bw.trailing();
    const int64_t nal = 1 + bw.pos;
    if (bw.overflow || nal + 4 > F.slot_cap) {
        F.lens[row] = -1;
        return;
    }
    slot[0] = (uint8_t)(nal >> 24); slot[1] = (uint8_t)(nal >> 16); slot[2] = (uint8_t)(nal >> 8); slot[3] = (uint8_t)nal;
    slot[4] = idr ? 0x65 : 0x61;             // nal_ref_idc 3, IDR slice / non-IDR slice
    F.lens[row] = (int32_t)(nal + 4);
}

// One block per row: offset = sum of the lengths of the rows above, then copy the slot.  The last row writes the sample length
// (-1 when any slot overflowed).
__global__ void __launch_bounds__(256) h264_pack(Frame F, uint8_t* sample, int64_t* sample_len) {
    __shared__ long long s_sum[8];
    __shared__ int s_bad[8];
    const int row = blockIdx.x, tid = threadIdx.x;
    long long off = 0;
    int bad = 0;
    for (int r = tid; r <= row; r += 256) {
        const int l = F.lens[r];
        if (l < 0) bad = 1;
        if (r < row) off += l;
    }
    for (int o = 16; o; o >>= 1) { off += __shfl_xor_sync(0xffffffffu, off, o); bad |= __shfl_xor_sync(0xffffffffu, bad, o); }
    if ((tid & 31) == 0) { s_sum[tid >> 5] = off; s_bad[tid >> 5] = bad; }
    __syncthreads();
    off = 0;
    bad = 0;
    for (int i = 0; i < 8; ++i) { off += s_sum[i]; bad |= s_bad[i]; }
    if (bad) {
        if (row == F.mbh - 1 && tid == 0) *sample_len = -1;
        return;
    }
    const int len = F.lens[row];
    const uint8_t* src = F.slots + row * F.slot_cap;
    for (int i = tid; i < len; i += 256) sample[off + i] = src[i];
    if (row == F.mbh - 1 && tid == 0) *sample_len = off + len;
}

int sizes(int width, int height, int64_t* plane_bytes, int64_t* scratch_bytes, int64_t* slot_cap, int64_t* slice_bytes) {
    N3D_CHECK_ARG(width > 0 && height > 0 && width % 2 == 0 && height % 2 == 0,
                  "n3d_h264: frame size %dx%d: 4:2:0 needs even, positive dimensions", width, height);
    const int64_t mbw = (width + 15) / 16, mbh = (height + 15) / 16;
    N3D_CHECK_ARG(mbw * mbh <= kMaxFs && mbw * mbw <= 8 * kMaxFs && mbh * mbh <= 8 * kMaxFs,
                  "n3d_h264: frame size %dx%d exceeds H.264 level 6.2 (%d macroblocks, at most %d per side)", width, height, kMaxFs, 1055);
    *plane_bytes = 256 * mbw * mbh * 3 / 2;
    *scratch_bytes = (int64_t)sizeof(MbRec) * mbw * mbh + 4 * mbh + 4 * (mbh + 1);     // MBs, slot lengths, deblocking counters
    // slot: 4-byte length, NAL header, escaped RBSP: slice header (<= 128 bits), MBs, trailing skip run and bits (<= 32 bits);
    // emulation prevention adds at most one byte per two
    const int64_t rbsp = (mbw * kMbBits + 128 + 32 + 7) / 8;
    *slot_cap = (5 + rbsp + rbsp / 2 + 1 + 15) / 16 * 16;
    *slice_bytes = *slot_cap * mbh;
    return N3D_OK;
}

}  // namespace

extern "C" int n3d_h264_buffer_sizes(int width, int height, int64_t* plane_bytes, int64_t* scratch_bytes, int64_t* slice_bytes,
                                     int64_t* sample_bytes) {
    N3D_CHECK_ARG(plane_bytes && scratch_bytes && slice_bytes && sample_bytes, "n3d_h264_buffer_sizes: null output pointer");
    int64_t cap;
    const int rc = sizes(width, height, plane_bytes, scratch_bytes, &cap, slice_bytes);
    if (rc != N3D_OK) return rc;
    *sample_bytes = *slice_bytes;
    return N3D_OK;
}

namespace {

// The kernels of one frame, in stream order; the rate-controlled stream adds the deblocking filter and the controller update.
template <bool kRc>
int launch(const char* name, const Frame& F, uint8_t* sample, int64_t* sample_len, cudaStream_t s) {
    h264_rgb_to_yuv<<<n3d_grid((int64_t)F.W16 * F.H16 / 4, 256), 256, 0, s>>>(F);
    if (F.idr) h264_intra_rows<kRc><<<F.mbh, 32, 0, s>>>(F);
    else h264_inter_mbs<kRc><<<dim3(F.mbw, F.mbh), 256, 0, s>>>(F);
    if constexpr (kRc) {
        const cudaError_t e = cudaMemsetAsync(F.dbk, 0, 4 * (F.mbh + 1), s);          // deblocking counters, per frame
        if (e != cudaSuccess) {
            n3d_set_error("%s: resetting the deblocking counters failed: %s", name, cudaGetErrorString(e));
            return N3D_ERR_CUDA;
        }
        h264_deblock<<<F.mbh, 32, 0, s>>>(F);
    }
    h264_write_rows<kRc><<<n3d_div_up(F.mbh, 32), 32, 0, s>>>(F);
    h264_pack<<<F.mbh, 256, 0, s>>>(F, sample, sample_len);
    if constexpr (kRc) h264_rc_update<<<1, 1, 0, s>>>(F.rc, sample_len, F.idr);
    N3D_CHECK_LAUNCH(name);
    return N3D_OK;
}

// Shared by both entry points: rc == nullptr runs the constant-QP stream at qp, else the rate-controlled stream.
int encode(const char* name, const uint8_t* rgb, int width, int height, int qp, int64_t* rc, int idr, int frame_num, int idr_pic_id,
           uint8_t* cur, const uint8_t* ref, uint8_t* recon, void* scratch, uint8_t* slices, uint8_t* sample, int64_t* sample_len,
           void* stream) {
    N3D_CHECK_ARG(rgb && cur && recon && scratch && slices && sample && sample_len, "%s: null buffer", name);
    N3D_CHECK_ARG(idr || ref, "%s: a P frame needs the reference reconstruction (null ref)", name);
    N3D_CHECK_ARG(ref != recon, "%s: ref and recon must be different buffers", name);
    N3D_CHECK_ARG(frame_num >= 0 && frame_num < 16 && idr_pic_id >= 0 && idr_pic_id <= 65535,
                  "%s: frame_num %d (0..15) or idr_pic_id %d (0..65535) out of range", name, frame_num, idr_pic_id);
    int64_t plane_bytes, scratch_bytes, slot_cap, slice_bytes;
    const int rc_ = sizes(width, height, &plane_bytes, &scratch_bytes, &slot_cap, &slice_bytes);
    if (rc_ != N3D_OK) return rc_;
    Frame F;
    F.W = width; F.H = height;
    F.mbw = (width + 15) / 16; F.mbh = (height + 15) / 16;
    F.W16 = 16 * F.mbw; F.H16 = 16 * F.mbh;
    F.qp = qp;
    F.rgb = rgb; F.cur = cur; F.ref = ref; F.rec = recon;
    F.mbs = (MbRec*)scratch;
    F.lens = (int32_t*)((uint8_t*)scratch + (int64_t)sizeof(MbRec) * F.mbw * F.mbh);
    F.dbk = F.lens + F.mbh;
    F.rc = rc;
    F.slots = slices; F.slot_cap = slot_cap;
    F.idr = idr ? 1 : 0; F.frame_num = frame_num; F.idr_pic_id = idr_pic_id;
    cudaStream_t s = (cudaStream_t)stream;
    return rc ? launch<true>(name, F, sample, sample_len, s) : launch<false>(name, F, sample, sample_len, s);
}

}  // namespace

extern "C" int n3d_h264_encode(const uint8_t* rgb, int width, int height, int qp, int idr, int frame_num, int idr_pic_id, uint8_t* cur,
                               const uint8_t* ref, uint8_t* recon, void* scratch, uint8_t* slices, uint8_t* sample, int64_t* sample_len,
                               void* stream) {
    N3D_CHECK_ARG(qp >= 0 && qp <= 51, "n3d_h264_encode: qp %d outside 0..51", qp);
    return encode("n3d_h264_encode", rgb, width, height, qp, nullptr, idr, frame_num, idr_pic_id, cur, ref, recon, scratch, slices, sample,
                  sample_len, stream);
}

extern "C" int n3d_h264_rc_init(void* state, int width, int height, int64_t bits_per_second, int fps_num, int fps_den, int qp_min,
                                int qp_max, void* stream) {
    N3D_CHECK_ARG(state, "n3d_h264_rc_init: null state");
    int64_t plane_bytes, scratch_bytes, slot_cap, slice_bytes;
    const int rc = sizes(width, height, &plane_bytes, &scratch_bytes, &slot_cap, &slice_bytes);
    if (rc != N3D_OK) return rc;
    N3D_CHECK_ARG(bits_per_second > 0 && bits_per_second <= 0xffffffffLL, "n3d_h264_rc_init: bits_per_second %lld outside 1..2^32-1",
                  (long long)bits_per_second);
    N3D_CHECK_ARG(fps_num > 0 && fps_den > 0 && fps_num <= (1 << 20) && fps_den <= (1 << 20),
                  "n3d_h264_rc_init: frame rate %d/%d: numerator and denominator must be in 1..2^20", fps_num, fps_den);
    N3D_CHECK_ARG(0 <= qp_min && qp_min <= qp_max && qp_max <= 51, "n3d_h264_rc_init: qp bounds %d..%d: need 0 <= qp_min <= qp_max <= 51",
                  qp_min, qp_max);
    h264_rc_init<<<1, 1, 0, (cudaStream_t)stream>>>((int64_t*)state, width, height, bits_per_second, fps_num, fps_den, qp_min, qp_max);
    N3D_CHECK_LAUNCH("n3d_h264_rc_init");
    return N3D_OK;
}

extern "C" int n3d_h264_encode_rc(const uint8_t* rgb, int width, int height, void* state, int idr, int frame_num, int idr_pic_id,
                                  uint8_t* cur, const uint8_t* ref, uint8_t* recon, void* scratch, uint8_t* slices, uint8_t* sample,
                                  int64_t* sample_len, void* stream) {
    N3D_CHECK_ARG(state, "n3d_h264_encode_rc: null state");
    return encode("n3d_h264_encode_rc", rgb, width, height, 0, (int64_t*)state, idr, frame_num, idr_pic_id, cur, ref, recon, scratch, slices,
                  sample, sample_len, stream);
}
