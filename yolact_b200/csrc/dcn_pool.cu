// Deformable position-sensitive RoI pooling (forward), fp32 NCHW.
//
// Reference: DeformablePSROIPoolForwardKernel and its bilinear_interp (external/DCNv2/src/cuda/
// dcn_v2_psroi_pooling_cuda.cu:33-146), restated here.  One thread per output element (r, ctop, ph, pw):
//   RoI      corners round()ed (half away from zero), * spatial_scale - 0.5, the end corner + 1; size max(.., 0.1)
//   bin      bin = size / pooled, sub-bin = bin / sample_per_part; part cell floor(ph / pooled * part_size);
//            class ctop / (output_dim / num_classes); start = p * bin + roi_start + trans * trans_std * size
//   channel  (ctop * group_size + gh) * group_size + gw, gh = clamp(floor(ph * group_size / pooled))
//   samples  sample_per_part^2 per bin; one outside [-0.5, W - 0.5] x [-0.5, H - 0.5] is skipped, the rest are clamped
//            to [0, W-1] x [0, H-1] and blended from the floor / ceil corners (which coincide on an integral position)
//   output   the mean of the counted samples, 0 when none was counted; count = the number counted
// Every fp32 product, sum and quotient is rounded on its own, in the order the reference's source writes it (no
// contraction into FMA), so that a restatement in any language reproduces the sampling positions bit for bit.
#include "kernels.cuh"

namespace yb {

namespace {

__global__ void __launch_bounds__(256) dcn_psroi_pool_kernel(const PsroiPoolArgs a) {
  const int P = a.pooled, gs = a.group_size, part = a.part_size, spp = a.sample_per_part;
  const int64_t total = (int64_t)a.R * a.output_dim * P * P;
  const int ceach = a.output_dim / a.num_classes;
  const float fP = (float)P;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int pw = (int)(idx % P);
    const int ph = (int)((idx / P) % P);
    const int ctop = (int)((idx / P / P) % a.output_dim);
    const int n = (int)(idx / P / P / a.output_dim);

    const float* roi = a.rois + (int64_t)n * 5;
    const int b = (int)__ldg(roi);   // checked on the host: finite, truncates into [0, N)
    const float s = a.spatial_scale;
    const float roi_start_w = __fsub_rn(__fmul_rn(roundf(__ldg(roi + 1)), s), 0.5f);
    const float roi_start_h = __fsub_rn(__fmul_rn(roundf(__ldg(roi + 2)), s), 0.5f);
    const float roi_end_w = __fsub_rn(__fmul_rn(__fadd_rn(roundf(__ldg(roi + 3)), 1.f), s), 0.5f);
    const float roi_end_h = __fsub_rn(__fmul_rn(__fadd_rn(roundf(__ldg(roi + 4)), 1.f), s), 0.5f);
    const float roi_w = fmaxf(__fsub_rn(roi_end_w, roi_start_w), 0.1f);   // fmax: a NaN size becomes 0.1, as there
    const float roi_h = fmaxf(__fsub_rn(roi_end_h, roi_start_h), 0.1f);
    const float bin_h = __fdiv_rn(roi_h, fP), bin_w = __fdiv_rn(roi_w, fP);
    const float sub_h = __fdiv_rn(bin_h, (float)spp), sub_w = __fdiv_rn(bin_w, (float)spp);

    float trans_x = 0.f, trans_y = 0.f;
    if (!a.no_trans) {
      const int part_h = (int)floorf(__fmul_rn(__fdiv_rn((float)ph, fP), (float)part));
      const int part_w = (int)floorf(__fmul_rn(__fdiv_rn((float)pw, fP), (float)part));
      const int cls = ctop / ceach;
      const float* t = a.trans + ((int64_t)n * a.num_classes + cls) * 2 * part * part + (int64_t)part_h * part + part_w;
      trans_x = __fmul_rn(__ldg(t), a.trans_std);
      trans_y = __fmul_rn(__ldg(t + (int64_t)part * part), a.trans_std);
    }
    const float wstart = __fadd_rn(__fadd_rn(__fmul_rn((float)pw, bin_w), roi_start_w), __fmul_rn(trans_x, roi_w));
    const float hstart = __fadd_rn(__fadd_rn(__fmul_rn((float)ph, bin_h), roi_start_h), __fmul_rn(trans_y, roi_h));

    const int gw = min(max((int)floorf(__fdiv_rn(__fmul_rn((float)pw, (float)gs), fP)), 0), gs - 1);
    const int gh = min(max((int)floorf(__fdiv_rn(__fmul_rn((float)ph, (float)gs), fP)), 0), gs - 1);
    const int c = (ctop * gs + gh) * gs + gw;
    const float* img = a.x + ((int64_t)b * a.C + c) * a.H * a.W;

    float sum = 0.f;
    int cnt = 0;
    for (int ih = 0; ih < spp; ++ih) {
      for (int iw = 0; iw < spp; ++iw) {
        float w = __fadd_rn(wstart, __fmul_rn((float)iw, sub_w));
        float h = __fadd_rn(hstart, __fmul_rn((float)ih, sub_h));
        if (w < -0.5f || w > (float)a.W - 0.5f || h < -0.5f || h > (float)a.H - 0.5f) continue;
        w = fminf(fmaxf(w, 0.f), (float)(a.W - 1));
        h = fminf(fmaxf(h, 0.f), (float)(a.H - 1));
        const int x1 = (int)floorf(w), x2 = (int)ceilf(w), y1 = (int)floorf(h), y2 = (int)ceilf(h);
        const float dx = __fsub_rn(w, (float)x1), dy = __fsub_rn(h, (float)y1);
        const float ux = __fsub_rn(1.f, dx), uy = __fsub_rn(1.f, dy);
        const float v11 = __ldg(img + (int64_t)y1 * a.W + x1), v12 = __ldg(img + (int64_t)y2 * a.W + x1);
        const float v21 = __ldg(img + (int64_t)y1 * a.W + x2), v22 = __ldg(img + (int64_t)y2 * a.W + x2);
        const float val = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(__fmul_rn(ux, uy), v11), __fmul_rn(__fmul_rn(ux, dy), v12)),
                                              __fmul_rn(__fmul_rn(dx, uy), v21)),
                                    __fmul_rn(__fmul_rn(dx, dy), v22));
        sum = __fadd_rn(sum, val);
        ++cnt;
      }
    }
    a.y[idx] = cnt == 0 ? 0.f : __fdiv_rn(sum, (float)cnt);
    if (a.count) a.count[idx] = (float)cnt;
  }
}

}  // namespace

void launch_dcn_psroi_pool(const PsroiPoolArgs& a, cudaStream_t stream, LaunchCounter* lc) {
  const int64_t total = (int64_t)a.R * a.output_dim * a.pooled * a.pooled;
  if (total == 0) return;
  const int blocks = (int)std::min<int64_t>((total + 255) / 256, 1 << 20);   // grid-stride beyond 2^28 elements
  dcn_psroi_pool_kernel<<<blocks, 256, 0, stream>>>(a);
  YB_CHECK_LAUNCH();
  if (lc) lc->n++;
}

}  // namespace yb
