// phisnet.cu -- PhiSNet's Clebsch-Gordan mixing layers (SURVEY.md section 8 f4).
//
// Replaces  PairMixing.forward      nablaDFT/phisnet/nn/modules/pair_mixing.py:47-69
//           SelfMixing.forward      nablaDFT/phisnet/nn/modules/self_mixing.py:55-83
//           SphericalLinear.forward nablaDFT/phisnet/nn/modules/spherical_linear.py:50-59 (per-order Linear: nb200_phis_linear)
// The reference loops over (l1, l2, L), forms the outer product x1 (x) x2 as a [.., 2l1+1, 2l2+1, 1, F] temporary, multiplies it with the
// broadcast CG tensor and sums twice: ~65 x 3 eager launches and a [P, 9, 9, 9, F] peak temporary per call.  Here features are stored
// component-major [rows][(L+1)^2][F] (channels contiguous), one thread owns one feature channel of one row, keeps a[25], b[25], o[25] in
// registers and evaluates the 2052 (pair) / 729 (self) non-zero real CG terms as unrolled FMAs (phisnet_cg_gen.inc, generated from the
// reference's vendored table).  SIMT on purpose: the CG tensors are > 80 % zeros; the dense work of the layer -- the distance-dependent
// coefficients rbf . W for all 65 paths, [P,128] x [128, 8320] -- runs on the wgmma 3xTF32 GEMM (nb200_dense) before this kernel.
#include "common.cuh"
#include "phisnet_cg_gen.inc"

namespace {

constexpr int PH_LM = 25;

// y[r][c][f] = sum_paths coeff[r][path][f] * CG : (x1[r] (x) x2[r])       coeff: [rows][n_paths][F] from the radial GEMM
__global__ void __launch_bounds__(128) k_phis_pair_mix(const float* __restrict__ x1, const float* __restrict__ x2, const float* __restrict__ coeff,
                                                      int n_paths, int o1, int o2, int oo, float* __restrict__ y) {
    const int r = blockIdx.x, f = threadIdx.x, F = blockDim.x;
    const int n1 = (o1 + 1) * (o1 + 1), n2 = (o2 + 1) * (o2 + 1), no = (oo + 1) * (oo + 1);
    float a[PH_LM], b[PH_LM], o[PH_LM];
#pragma unroll
    for (int k = 0; k < PH_LM; ++k) {
        a[k] = k < n1 ? __ldg(x1 + ((size_t)r * n1 + k) * F + f) : 0.f;
        b[k] = k < n2 ? __ldg(x2 + ((size_t)r * n2 + k) * F + f) : 0.f;
        o[k] = 0.f;
    }
    phis_pair_couple(a, b, coeff + (size_t)r * n_paths * F + f, F, o1, o2, oo, o);
#pragma unroll
    for (int k = 0; k < PH_LM; ++k)
        if (k < no) y[((size_t)r * no + k) * F + f] = o[k];
}

// y[r][c][f] = keep[L(c)][f] x[r][c][f] + sum_{l1<l2} mix[path][f] * CG : (x[r] (x) x[r])
__global__ void __launch_bounds__(128) k_phis_self_mix(const float* __restrict__ x, const float* __restrict__ mix, const float* __restrict__ keep, int oi,
                                                      int oo, float* __restrict__ y) {
    const int r = blockIdx.x, f = threadIdx.x, F = blockDim.x;
    const int ni = (oi + 1) * (oi + 1), no = (oo + 1) * (oo + 1);
    float a[PH_LM], o[PH_LM];
#pragma unroll
    for (int k = 0; k < PH_LM; ++k) a[k] = k < ni ? __ldg(x + ((size_t)r * ni + k) * F + f) : 0.f;
#pragma unroll
    for (int L = 0; L < 5; ++L) {
        const float kc = (L <= oi && L <= oo) ? __ldg(keep + (size_t)L * F + f) : 0.f;
#pragma unroll
        for (int m = 0; m < 2 * L + 1; ++m) o[L * L + m] = kc * a[L * L + m];
    }
    phis_self_couple(a, a, mix + f, F, oi, oi, oo, o);
#pragma unroll
    for (int k = 0; k < PH_LM; ++k)
        if (k < no) y[((size_t)r * no + k) * F + f] = o[k];
}

bool feat_ok(int F) { return F == 32 || F == 64 || F == 96 || F == 128; }
bool order_ok(int o) { return o >= 0 && o <= 4; }

}  // namespace

extern "C" int nb200_phis_n_paths(int32_t order_in1, int32_t order_in2, int32_t order_out, int32_t strict_upper) {
    if (!order_ok(order_in1) || !order_ok(order_in2) || !order_ok(order_out)) return NB200_EINVAL;
    int n = 0;
    for (int l1 = 0; l1 <= order_in1; ++l1)
        for (int l2 = strict_upper ? l1 + 1 : 0; l2 <= order_in2; ++l2)
            for (int L = (l1 > l2 ? l1 - l2 : l2 - l1); L <= (l1 + l2 < order_out ? l1 + l2 : order_out); ++L) ++n;
    return n;
}

extern "C" int nb200_phis_pair_mixing(const float* x1, const float* x2, const float* coeff, int32_t n_rows, int32_t n_feat, int32_t order_in1,
                                      int32_t order_in2, int32_t order_out, float* y, void* stream) {
    if (!x1 || !x2 || !coeff || !y || n_rows < 0) return NB200_EINVAL;
    if (!feat_ok(n_feat) || !order_ok(order_in1) || !order_ok(order_in2) || !order_ok(order_out)) return NB200_EUNSUPPORTED;
    if (n_rows == 0) return NB200_OK;
    const int n_paths = nb200_phis_n_paths(order_in1, order_in2, order_out, 0);
    k_phis_pair_mix<<<n_rows, n_feat, 0, (cudaStream_t)stream>>>(x1, x2, coeff, n_paths, order_in1, order_in2, order_out, y);
    return nb_check_launch();
}

extern "C" int nb200_phis_self_mixing(const float* x, const float* mixcoeff, const float* keepcoeff, int32_t n_rows, int32_t n_feat, int32_t order_in,
                                      int32_t order_out, float* y, void* stream) {
    if (!x || !mixcoeff || !keepcoeff || !y || n_rows < 0) return NB200_EINVAL;
    if (!feat_ok(n_feat) || !order_ok(order_in) || !order_ok(order_out)) return NB200_EUNSUPPORTED;
    if (n_rows == 0) return NB200_OK;
    k_phis_self_mix<<<n_rows, n_feat, 0, (cudaStream_t)stream>>>(x, mixcoeff, keepcoeff, order_in, order_out, y);
    return nb_check_launch();
}

// per-order Linear over component-major features: y[r][c][:] = x[r][c][:] . W_{L(c)} (+ bias on c = 0).  W_l: [order+1][c_in][c_out].
extern "C" int nb200_phis_linear(const float* x, const float* W_l, const float* bias, int32_t n_rows, int32_t c_in, int32_t c_out, int32_t order,
                                 float* y, void* stream) {
    if (!x || !W_l || !y || !order_ok(order)) return NB200_EINVAL;
    const int nc = (order + 1) * (order + 1);
    return nb_gemm_tf32x3_lm(n_rows, c_out, c_in, x, nc * c_in, W_l, (long long)c_in * c_out, y, nc * c_out, 0, bias, nc, (cudaStream_t)stream);
}
