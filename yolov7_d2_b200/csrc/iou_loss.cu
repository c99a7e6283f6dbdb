// Box-regression losses on matched (prediction, target) pairs with their gradient w.r.t. the prediction:
//   mode 0  IOUloss "iou"   1 - iou^2                       yolov7/utils/boxes.py:125-151   (YOLOX head, yolox_head.py:134)
//   mode 1  IOUloss "giou"  1 - clamp(giou, -1, 1)          boxes.py:152-161
//   mode 2  IOUlossV6 giou  mode 3 diou  mode 4 ciou        boxes.py:666-752                 (YOLOv6 head; the north star's "CIoU")
// Boxes are (cx, cy, w, h); the gradient comes from the dual numbers of dual4.cuh, so the kernel text follows the reference formula line by
// line (including which epsilons are added where and the detached alpha of CIoU).
#include "dual4.cuh"
#include "host_common.cuh"
#include "sm90.cuh"

using namespace yb;

namespace {

__global__ void iou_loss_kernel(const float* __restrict__ pred, const float* __restrict__ tgt, int n, int mode, float* __restrict__ loss,
                                float* __restrict__ dpred) {
  pdl_sync();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const D4 px = var(pred[4 * i], 0), py = var(pred[4 * i + 1], 1), pw = var(pred[4 * i + 2], 2), ph = var(pred[4 * i + 3], 3);
  const D4 tx = cst(tgt[4 * i]), ty = cst(tgt[4 * i + 1]), tw = cst(tgt[4 * i + 2]), th = cst(tgt[4 * i + 3]);
  const D4 p_l = px - pw * 0.5f, p_r = px + pw * 0.5f, p_t = py - ph * 0.5f, p_b = py + ph * 0.5f;
  const D4 t_l = tx - tw * 0.5f, t_r = tx + tw * 0.5f, t_t = ty - th * 0.5f, t_b = ty + th * 0.5f;
  D4 l;
  if (mode <= 1) {
    // IOUloss (boxes.py:131-161)
    const D4 tlx = dmax(p_l, t_l), tly = dmax(p_t, t_t), brx = dmin(p_r, t_r), bry = dmin(p_b, t_b);
    const float en = (tlx.v < brx.v && tly.v < bry.v) ? 1.f : 0.f;
    const D4 area_i = (brx - tlx) * (bry - tly) * en;
    const D4 area_p = pw * ph, area_g = tw * th;
    const D4 iou = area_i / (area_p + area_g - area_i + 1e-16f);
    if (mode == 0) {
      l = 1.f - iou * iou;
    } else {
      const D4 c_tlx = dmin(p_l, t_l), c_tly = dmin(p_t, t_t), c_brx = dmax(p_r, t_r), c_bry = dmax(p_b, t_b);
      const D4 area_c = (c_brx - c_tlx) * (c_bry - c_tly);
      const D4 giou = iou - (area_c - area_i) / clamp_min(area_c, 1e-16f);
      l = 1.f - clamp(giou, -1.f, 1.f);
    }
  } else {
    // IOUlossV6, box_format "xywh" (boxes.py:696-733), eps = 1e-7
    const float eps = 1e-7f;
    const D4 inter = clamp_min(dmin(p_r, t_r) - dmax(p_l, t_l), 0.f) * clamp_min(dmin(p_b, t_b) - dmax(p_t, t_t), 0.f);
    const D4 w1 = p_r - p_l, h1 = p_b - p_t + eps, w2 = t_r - t_l, h2 = t_b - t_t + eps;
    const D4 uni = w1 * h1 + w2 * h2 - inter + eps;
    D4 iou = inter / uni;
    const D4 cw = dmax(p_r, t_r) - dmin(p_l, t_l), ch = dmax(p_b, t_b) - dmin(p_t, t_t);
    if (mode == 2) {
      const D4 c_area = cw * ch + eps;
      iou = iou - (c_area - uni) / c_area;
    } else {
      const D4 c2 = cw * cw + ch * ch + eps;
      const D4 dx = t_l + t_r - p_l - p_r, dy = t_t + t_b - p_t - p_b;
      const D4 rho2 = (dx * dx + dy * dy) * 0.25f;
      if (mode == 3) {
        iou = iou - rho2 / c2;
      } else {
        const D4 da = datan(w2 / h2) - datan(w1 / h1);
        const D4 v = da * da * (4.f / (3.14159265358979323846f * 3.14159265358979323846f));
        const float alpha = v.v / (v.v - iou.v + (1.f + eps));  // computed under torch.no_grad(): a constant
        iou = iou - (rho2 / c2 + v * alpha);
      }
    }
    l = 1.f - iou;
  }
  loss[i] = l.v;
  if (dpred) {
    dpred[4 * i] = l.g[0];
    dpred[4 * i + 1] = l.g[1];
    dpred[4 * i + 2] = l.g[2];
    dpred[4 * i + 3] = l.g[3];
  }
}

}  // namespace

extern "C" int yb200_iou_loss(const float* pred_cxcywh, const float* target_cxcywh, int n, int mode, float* loss, float* dloss_dpred,
                              void* stream) {
  YB_REQUIRE(pred_cxcywh && target_cxcywh && loss, YB200_ERR_INVALID, "iou_loss: null pointer");
  YB_REQUIRE(n >= 0 && mode >= 0 && mode <= 4, YB200_ERR_INVALID, "iou_loss: n=%d mode=%d", n, mode);
  if (n == 0) return 0;
  launch_k(iou_loss_kernel, ceil_div(n, 128), 128, 0, as_stream(stream), pred_cxcywh, target_cxcywh, n, mode, loss, dloss_dpred);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
