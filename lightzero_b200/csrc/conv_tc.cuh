// conv_tc.cuh -- wgmma 3x3 convolutions of the DownSample tower (representation network).
//
// Activations between tower layers live in HBM in a tensor-core-ready layout ("TCL"): per image
//   [part: fp16 hi | fp16 lo][k-group of 8 channels][row][8 halves]
// where `row` walks a zero-padded grid of pitch W+1 (one pad column) with one pad row above and below:
//   rho = (y + 1) * pitch + x,   memory row = rho + 1   (one spare zero row at each end),
//   rows per plane R = (H + 2) * pitch + 2.
// A band of image rows is then a handful of contiguous cp.async.bulk copies per plane, lands in shared
// memory already in the wgmma K-major / no-swizzle canonical layout, and every 3x3 tap is the same buffer
// read through a row-shifted descriptor (see net_tc.cu).  Stride-2 convolutions read a 4-phase
// (space-to-depth) variant written by the producing layer: phase (y&1, x&1) image of half size, so that
// tap (ky,kx) is phase ((ky+1)&1, (kx+1)&1) shifted by (ky==0 ? -1 : 0, kx==0 ? -1 : 0).
#pragma once
#include "lz_common.cuh"

namespace lz {

struct Tcl {                      // one activation tensor in TCL
    unsigned char *base;
    size_t img_stride, phase_stride, part_stride;   // bytes
    int plane_rows;               // R (rows per k-group plane, incl. the 2 spare rows)
    int C, H, W, pitch;           // geometry of ONE phase image (== the tensor itself when nphase == 1)
    int nphase;                   // 1 or 4
};

inline Tcl make_tcl(unsigned char *base, int C, int H, int W, int nphase)
{
    Tcl t;
    t.base = base; t.C = C; t.H = H; t.W = W; t.pitch = W + 1; t.nphase = nphase;
    t.plane_rows = (H + 2) * (W + 1) + 2;
    t.part_stride = (size_t)(C / 8) * t.plane_rows * 16;
    t.phase_stride = 2 * t.part_stride;
    t.img_stride = t.phase_stride * nphase;
    return t;
}
inline size_t tcl_bytes(int B, int C, int H, int W, int nphase)
{
    return (size_t)B * nphase * 2 * (C / 8) * ((size_t)(H + 2) * (W + 1) + 2) * 16;
}

struct ConvTc {
    Tcl in;                       // input (nphase 1 or 4); its (H, W, pitch) is the output/row-space geometry
    Tcl out[2];                   // column group 0 / 1 (group 1 only for N = 128), nphase 1
    Tcl res;                      // residual added to group 0 (base == nullptr: none)
    const unsigned char *w;       // [9 taps][kg_in][N hi rows | N lo rows][8] fp16
    const float *scale, *shift;   // [N]
    int tap_phase[9], tap_shift[9];
    int relu[2];
    int N;                        // 64 or 128
    int G, band_h;                // images per CTA (band_h == H when G > 1), image rows per band
    int stages;                   // weight ring depth (2..4)
    int B, npass;
};

// One plain ResBlock, relu(bn2(conv2(relu(bn1(conv1(x))))) + x), C -> C channels at stride 1, in one kernel: conv1's output
// stays in shared memory (see k_resblock_tc)
struct ResBlockTc {
    Tcl in;                       // x (nphase 1); its (C, H, W, pitch) is the geometry of the whole block
    Tcl out;                      // nphase 1, or 4 = written phase-split for a stride-2 consumer
    const unsigned char *w[2];    // conv1 / conv2 tap blocks (conv_tc_pack with ncols = C)
    const float *scale[2], *shift[2];
    int tap_shift[9];
    int G, band_h;                // images per CTA (band_h == H when G > 1), output rows per band
    int stages;                   // weight ring depth (2 or 4)
    int B, npass;
};

int conv_tc_prepare_launch();
int conv_tc_launch(const ConvTc &p, cudaStream_t s);
// picks G, band_h and stages of a ResBlockTc whose `in` geometry is set; returns LZ_EINVAL if no band fits
int resblock_tc_plan(ResBlockTc &p);
int resblock_tc_launch(const ResBlockTc &p, cudaStream_t s);
// weights [cout][cin][3][3] -> tap blocks with `ncols` columns, this tensor occupying columns
// [col0, col0+cout); returns the exact power-of-two scale applied
float conv_tc_pack(const float *w_torch, int cin, int cout, int ncols, int col0, unsigned char *dst);
size_t conv_tc_packed_bytes(int cin, int ncols);

// pooling on TCL tensors: AvgPool2d(3, stride 2, pad 1), count_include_pad -> /9
int pool_tcl_launch(const Tcl &in, const Tcl &out, int B, cudaStream_t s);                 // TCL -> TCL
int pool_tcl_to_nchw_launch(const Tcl &in, float *out, int B, int Hout, cudaStream_t s);   // TCL -> fp32 NCHW
// TCL -> fp32 NCHW at the same size (hi + lo; the 64-pixel tower's last step), and the CTAs that launch uses
int tcl_to_nchw_launch(const Tcl &in, float *out, int B, cudaStream_t s);
int tcl_to_nchw_ctas(const Tcl &in, int B);

}  // namespace lz
