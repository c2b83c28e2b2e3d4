// SIMT fp32 implicit-GEMM convolution on NHWC activations (exact fp32 FMA accumulation).
//
// This is the reference-accuracy engine: every dense conv of the path can run here, and the small-channel /
// HBM-bound layers (3-, 8-, 24-, 72-channel convs) always do.  The big GEMM-shaped layers move to the wgmma
// engine (conv2d_tc.cu) once that is parity-green against this kernel.
//
//   M = B*Ho*Wo output pixels, N = Cout, K = KH*KW*Cin.   CTA tile 128 x BN, K-chunk 16, 256 threads,
//   register tile 8 x (BN/16), gmem->register prefetch of the next chunk overlapped with the FMA loop.
//   BN + ReLU + residual + channel-slice (concat) write fused in the epilogue.
#include "common.cuh"

namespace vd3d {

constexpr int CBM = 128;
constexpr int CBK = 16;
constexpr int CTHREADS = 256;

struct ConvParams {
    const float* in; const float* wgt; const float* bias; const float* res; float* out;
    int B, H, W, Cin, in_cs, in_co;
    int KH, KW, stride, pad, dil;
    int Ho, Wo, Cout, out_cs, out_co, res_cs, res_co;
    int relu;
    int M, K;
};

template <int BN, int VEC>
__global__ void __launch_bounds__(CTHREADS) conv2d_simt_kernel(const ConvParams p) {
    constexpr int TN = BN / 16;
    constexpr int APAD = 4;
    __shared__ __align__(16) float As[CBK][CBM + APAD];
    __shared__ __align__(16) float Bs[CBK][BN];

    const int t = threadIdx.x;
    const int m0 = blockIdx.x * CBM;
    const int n0 = blockIdx.y * BN;
    const int tx = t & 15, ty = t >> 4;

    // ---- A-load bookkeeping -------------------------------------------------------------------------------
    // VEC==4: thread loads 2 float4: rows (t>>2) and (t>>2)+64, k-quad (t&3)
    // VEC==1: thread loads 8 scalars: row (t&127), k = (t>>7) + 2*j
    constexpr int NA = (VEC == 4) ? 2 : 8;
    int a_hb[2], a_wb[2];            // top-left input coordinate of the 2 pixels this thread gathers (VEC 4)
    long long a_base[2];
    bool a_ok[2];
    {
        const int nrows = (VEC == 4) ? 2 : 1;
#pragma unroll
        for (int j = 0; j < nrows; ++j) {
            int m = m0 + ((VEC == 4) ? ((t >> 2) + 64 * j) : (t & 127));
            a_ok[j] = m < p.M;
            int mm = a_ok[j] ? m : 0;
            int wo = mm % p.Wo; int r = mm / p.Wo; int ho = r % p.Ho; int b = r / p.Ho;
            a_hb[j] = ho * p.stride - p.pad;
            a_wb[j] = wo * p.stride - p.pad;
            a_base[j] = (long long)b * p.H * p.W;
        }
        if (VEC != 4) { a_hb[1] = a_hb[0]; a_wb[1] = a_wb[0]; a_base[1] = a_base[0]; a_ok[1] = a_ok[0]; }
    }
    // ---- B-load bookkeeping: BK x BN floats = 4*BN float4 --------------------------------------------------
    constexpr int NB4 = (CBK * BN / 4 + CTHREADS - 1) / CTHREADS;   // float4 per thread
    constexpr int BCOLS4 = BN / 4;

    float4 ra[(VEC == 4) ? 2 : 1];
    float ras[(VEC == 4) ? 1 : 8];
    float4 rb[NB4];

    auto load_chunk = [&](int k0) {
        if (VEC == 4) {
            int k = k0 + 4 * (t & 3);
            int tap = k / p.Cin; int ci = k - tap * p.Cin;
            int kh = tap / p.KW; int kw = tap - kh * p.KW;
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                int hi = a_hb[j] + kh * p.dil, wi = a_wb[j] + kw * p.dil;
                bool ok = a_ok[j] && k < p.K && hi >= 0 && hi < p.H && wi >= 0 && wi < p.W;
                ra[j] = ok ? ldg4(p.in + (a_base[j] + (long long)hi * p.W + wi) * p.in_cs + p.in_co + ci)
                           : make_float4(0.f, 0.f, 0.f, 0.f);
            }
        } else {
#pragma unroll
            for (int j = 0; j < NA; ++j) {
                int k = k0 + (t >> 7) + 2 * j;
                int tap = k / p.Cin; int ci = k - tap * p.Cin;
                int kh = tap / p.KW; int kw = tap - kh * p.KW;
                int hi = a_hb[0] + kh * p.dil, wi = a_wb[0] + kw * p.dil;
                bool ok = a_ok[0] && k < p.K && hi >= 0 && hi < p.H && wi >= 0 && wi < p.W;
                ras[j] = ok ? __ldg(p.in + (a_base[0] + (long long)hi * p.W + wi) * p.in_cs + p.in_co + ci) : 0.f;
            }
        }
#pragma unroll
        for (int j = 0; j < NB4; ++j) {
            int idx = t + j * CTHREADS;
            int kr = idx / BCOLS4, c4 = idx - kr * BCOLS4;
            int k = k0 + kr, n = n0 + 4 * c4;
            bool ok = (idx < CBK * BCOLS4) && k < p.K && n < p.Cout;
            rb[j] = ok ? ldg4(p.wgt + (long long)k * p.Cout + n) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    };
    auto store_chunk = [&]() {
        if (VEC == 4) {
            int kq = 4 * (t & 3);
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                int r = (t >> 2) + 64 * j;
                As[kq + 0][r] = ra[j].x; As[kq + 1][r] = ra[j].y; As[kq + 2][r] = ra[j].z; As[kq + 3][r] = ra[j].w;
            }
        } else {
#pragma unroll
            for (int j = 0; j < NA; ++j) As[(t >> 7) + 2 * j][t & 127] = ras[j];
        }
#pragma unroll
        for (int j = 0; j < NB4; ++j) {
            int idx = t + j * CTHREADS;
            if (idx < CBK * BCOLS4) {
                int kr = idx / BCOLS4, c4 = idx - kr * BCOLS4;
                *reinterpret_cast<float4*>(&Bs[kr][4 * c4]) = rb[j];
            }
        }
    };

    float acc[8][TN];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

    const int nchunks = (p.K + CBK - 1) / CBK;
    load_chunk(0);
    for (int c = 0; c < nchunks; ++c) {
        store_chunk();
        __syncthreads();
        if (c + 1 < nchunks) load_chunk((c + 1) * CBK);
#pragma unroll
        for (int k = 0; k < CBK; ++k) {
            float a[8], b[TN];
            float4 a0 = *reinterpret_cast<const float4*>(&As[k][ty * 8]);
            float4 a1 = *reinterpret_cast<const float4*>(&As[k][ty * 8 + 4]);
            a[0] = a0.x; a[1] = a0.y; a[2] = a0.z; a[3] = a0.w; a[4] = a1.x; a[5] = a1.y; a[6] = a1.z; a[7] = a1.w;
            if (TN >= 4) {
#pragma unroll
                for (int j = 0; j < TN; j += 4) {
                    float4 bv = *reinterpret_cast<const float4*>(&Bs[k][tx * TN + j]);
                    b[j] = bv.x; b[j + 1] = bv.y; b[j + 2] = bv.z; b[j + 3] = bv.w;
                }
            } else {
#pragma unroll
                for (int j = 0; j < TN; ++j) b[j] = Bs[k][tx * TN + j];
            }
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }

    // ---- epilogue: bias (+residual) (+ReLU), channel-slice store ------------------------------------------
    float bj[TN];
#pragma unroll
    for (int j = 0; j < TN; ++j) {
        int n = n0 + tx * TN + j;
        bj[j] = (p.bias != nullptr && n < p.Cout) ? __ldg(p.bias + n) : 0.f;
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        int m = m0 + ty * 8 + i;
        if (m >= p.M) continue;
        float* op = p.out + (long long)m * p.out_cs + p.out_co;
        const float* rp = p.res ? p.res + (long long)m * p.res_cs + p.res_co : nullptr;
#pragma unroll
        for (int j = 0; j < TN; ++j) {
            int n = n0 + tx * TN + j;
            if (n < p.Cout) {
                float v = acc[i][j] + bj[j];
                if (rp) v += __ldg(rp + n);
                if (p.relu) v = fmaxf(v, 0.f);
                acc[i][j] = v;
            }
        }
        if (TN % 4 == 0) {
#pragma unroll
            for (int j = 0; j < TN; j += 4) {
                int n = n0 + tx * TN + j;
                if (n < p.Cout) *reinterpret_cast<float4*>(op + n) = make_float4(acc[i][j], acc[i][j + 1], acc[i][j + 2], acc[i][j + 3]);
            }
        } else {
#pragma unroll
            for (int j = 0; j < TN; ++j) {
                int n = n0 + tx * TN + j;
                if (n < p.Cout) op[n] = acc[i][j];
            }
        }
    }
}

template <int BN, int VEC>
static int launch_conv(const ConvParams& p, cudaStream_t st) {
    dim3 grid(cdiv(p.M, CBM), cdiv(p.Cout, BN));
    conv2d_simt_kernel<BN, VEC><<<grid, CTHREADS, 0, st>>>(p);
    VD3D_CHECK_LAUNCH("conv2d_simt");
    return VD3D_OK;
}

}  // namespace vd3d

using namespace vd3d;

extern "C" int vd3d_conv2d_nhwc(const float* in, int B, int H, int W, int Cin, int in_cs, int in_co,
                                const float* wgt, const float* bias, int KH, int KW, int stride, int pad, int dil,
                                const float* res, int res_cs, int res_co,
                                float* out, int Cout, int out_cs, int out_co, int relu, void* stream) {
    VD3D_REQUIRE(in && wgt && out, "conv2d: null pointer");
    VD3D_REQUIRE(B > 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0, "conv2d: bad shape");
    VD3D_REQUIRE(Cout % 4 == 0 && out_cs % 4 == 0 && out_co % 4 == 0, "conv2d: Cout/out pitch/offset must be multiples of 4 (Cout=%d cs=%d co=%d)", Cout, out_cs, out_co);
    VD3D_REQUIRE(!res || (res_cs % 4 == 0 && res_co % 4 == 0), "conv2d: residual pitch/offset must be multiples of 4");
    VD3D_REQUIRE(stride >= 1 && dil >= 1 && pad >= 0 && KH >= 1 && KW >= 1, "conv2d: bad conv params");
    ConvParams p;
    p.in = in; p.wgt = wgt; p.bias = bias; p.res = res; p.out = out;
    p.B = B; p.H = H; p.W = W; p.Cin = Cin; p.in_cs = in_cs; p.in_co = in_co;
    p.KH = KH; p.KW = KW; p.stride = stride; p.pad = pad; p.dil = dil;
    p.Ho = (H + 2 * pad - dil * (KH - 1) - 1) / stride + 1;
    p.Wo = (W + 2 * pad - dil * (KW - 1) - 1) / stride + 1;
    VD3D_REQUIRE(p.Ho > 0 && p.Wo > 0, "conv2d: empty output");
    p.Cout = Cout; p.out_cs = out_cs; p.out_co = out_co; p.res_cs = res_cs; p.res_co = res_co; p.relu = relu;
    long long M = (long long)B * p.Ho * p.Wo;
    VD3D_REQUIRE(M < (1ll << 31), "conv2d: too many output pixels");
    p.M = (int)M; p.K = KH * KW * Cin;
    cudaStream_t st = (cudaStream_t)stream;
    bool vec = (Cin % 4 == 0) && (in_cs % 4 == 0) && (in_co % 4 == 0) && ((reinterpret_cast<uintptr_t>(in) & 15) == 0);
    if (vec) {
        if (Cout > 64) return launch_conv<128, 4>(p, st);
        if (Cout > 32) return launch_conv<64, 4>(p, st);
        if (Cout > 16) return launch_conv<32, 4>(p, st);
        return launch_conv<16, 4>(p, st);
    } else {
        if (Cout > 64) return launch_conv<128, 1>(p, st);
        if (Cout > 32) return launch_conv<64, 1>(p, st);
        if (Cout > 16) return launch_conv<32, 1>(p, st);
        return launch_conv<16, 1>(p, st);
    }
}
