// TensorFlow custom-op registration shim over the bts_b200 C ABI (SURVEY 8f rank 4, "TF-op surface").
//
// Re-exposes the sm_90a LPG kernels behind the op names / signatures the reference's TF graph code binds:
//   lpg.local_planar_guidance(plane_eq, upratio=r, focal=...)        tensorflow/bts.py:279,294,309
//   lpg.local_planar_guidance_grad(depth_grad, input, focal)         tensorflow/custom_layer/_local_planar_guidance_grad.py:33
// i.e. ops "LocalPlanarGuidance" (input: float[B,h,w,4], focal: float[B], attr upratio:int -> depth: float[B,h*r,w*r]) and
// "LocalPlanarGuidanceGrad" (depth_grad, input, focal -> grad_input, grad_focal), the interface declared at
// tensorflow/custom_layer/local_planar_guidance.cc:67-72,234-239.  The bodies below are ours: each Compute() forwards raw
// device pointers + the op's CUDA stream to bts_lpg_fwd / bts_lpg_bwd (include/bts_b200.h) with layout = NHWC and
// tf_compat = 1 (the reference's TF gradient omits the factor n4 on dn1..dn3 -- SURVEY Q5 -- which a drop-in must keep).
// Differences by design: no per-launch device synchronisation (the reference calls d.synchronize() after every launch,
// local_planar_guidance.cu:91,170), grad_focal is written as zeros (the reference leaves it unset on CPU and aliases it to
// `focal` on GPU, .cc:326-329,391-393; `focal` never enters the arithmetic, SURVEY Q1).
//
// Build (where TensorFlow is installed; it is NOT in this image, so this file is not part of __graft_entry__.build()):
//   g++ -std=c++17 -shared -fPIC bts_lpg_tf_op.cc -o liblpg.so -I<repo>/include \
//       $(python -c 'import tensorflow as tf; print(" ".join(tf.sysconfig.get_compile_flags()))') \
//       $(python -c 'import tensorflow as tf; print(" ".join(tf.sysconfig.get_link_flags()))') \
//       -L<repo>/bts_b200 -lbts_b200 -Wl,-rpath,<repo>/bts_b200 -DGOOGLE_CUDA=1
// Then `tf.load_op_library('.../liblpg.so')` exactly as tensorflow/bts.py:29 does.
#include "tensorflow/core/framework/op.h"
#include "tensorflow/core/framework/op_kernel.h"
#include "tensorflow/core/framework/shape_inference.h"

#include "bts_b200.h"

namespace bts_b200_tf {

using namespace tensorflow;  // NOLINT

static Status LpgShape(shape_inference::InferenceContext *c) {
    shape_inference::ShapeHandle in;
    TF_RETURN_IF_ERROR(c->WithRank(c->input(0), 4, &in));
    int r = 0;
    TF_RETURN_IF_ERROR(c->GetAttr("upratio", &r));
    if (r < 1 || (r > 1 && (r & 1))) return errors::InvalidArgument("upratio must be 1 or even, got ", r);
    shape_inference::DimensionHandle h, w;
    TF_RETURN_IF_ERROR(c->Multiply(c->Dim(in, 1), r, &h));
    TF_RETURN_IF_ERROR(c->Multiply(c->Dim(in, 2), r, &w));
    c->set_output(0, c->MakeShape({c->Dim(in, 0), h, w}));
    return Status();
}

REGISTER_OP("LocalPlanarGuidance")
    .Input("input: float")
    .Input("focal: float")
    .Output("depth: float")
    .Attr("upratio: int")
    .SetShapeFn(LpgShape);

REGISTER_OP("LocalPlanarGuidanceGrad")
    .Input("depth_grad: float")
    .Input("input: float")
    .Input("focal: float")
    .Output("grad_input: float")
    .Output("grad_focal: float");

// device pointers in, asynchronous launch on the op's stream (GPU) or the host entry points (CPU placement)
template <bool kGpu>
class LpgOp : public OpKernel {
 public:
    explicit LpgOp(OpKernelConstruction *ctx) : OpKernel(ctx) { OP_REQUIRES_OK(ctx, ctx->GetAttr("upratio", &r_)); }
    void Compute(OpKernelContext *ctx) override {
        const Tensor &in = ctx->input(0);
        OP_REQUIRES(ctx, in.dims() == 4 && in.dim_size(3) == 4, errors::InvalidArgument("input must be [B,h,w,4]"));
        const int B = in.dim_size(0), h = in.dim_size(1), w = in.dim_size(2);
        Tensor *out = nullptr;
        OP_REQUIRES_OK(ctx, ctx->allocate_output(0, TensorShape({B, (int64_t)h * r_, (int64_t)w * r_}), &out));
        int rc;
        if (kGpu) {
            void *stream = *reinterpret_cast<void *const *>(ctx->op_device_context()->stream()->platform_specific_handle().stream);
            rc = bts_lpg_fwd(in.flat<float>().data(), out->flat<float>().data(), B, h, w, r_, BTS_LAYOUT_NHWC, stream);
        } else {
            rc = bts_lpg_fwd_h(in.flat<float>().data(), out->flat<float>().data(), B, h, w, r_, BTS_LAYOUT_NHWC);
        }
        OP_REQUIRES(ctx, rc == 0, errors::Internal("bts_lpg_fwd failed with code ", rc));
    }

 private:
    int r_ = 1;
};

template <bool kGpu>
class LpgGradOp : public OpKernel {
 public:
    explicit LpgGradOp(OpKernelConstruction *ctx) : OpKernel(ctx) {}
    void Compute(OpKernelContext *ctx) override {
        const Tensor &dy = ctx->input(0), &in = ctx->input(1), &focal = ctx->input(2);
        OP_REQUIRES(ctx, in.dims() == 4 && in.dim_size(3) == 4 && dy.dims() == 3,
                    errors::InvalidArgument("expected depth_grad [B,H,W] and input [B,h,w,4]"));
        const int B = in.dim_size(0), h = in.dim_size(1), w = in.dim_size(2);
        OP_REQUIRES(ctx, h > 0 && dy.dim_size(1) % h == 0, errors::InvalidArgument("depth_grad / input shape mismatch"));
        const int r = dy.dim_size(1) / h;
        Tensor *gin = nullptr, *gfocal = nullptr;
        OP_REQUIRES_OK(ctx, ctx->allocate_output(0, in.shape(), &gin));
        OP_REQUIRES_OK(ctx, ctx->allocate_output(1, focal.shape(), &gfocal));
        int rc;
        if (kGpu) {
            void *stream = *reinterpret_cast<void *const *>(ctx->op_device_context()->stream()->platform_specific_handle().stream);
            rc = bts_lpg_bwd(dy.flat<float>().data(), in.flat<float>().data(), gin->flat<float>().data(), B, h, w, r,
                             BTS_LAYOUT_NHWC, /*tf_compat=*/1, stream);
            if (rc == 0) rc = bts_fill_zero_f32(gfocal->flat<float>().data(), focal.NumElements(), stream);
        } else {
            rc = bts_lpg_bwd_h(dy.flat<float>().data(), in.flat<float>().data(), gin->flat<float>().data(), B, h, w, r,
                               BTS_LAYOUT_NHWC, 1);
            float *gf = gfocal->flat<float>().data();
            for (int64_t i = 0; i < focal.NumElements(); ++i) gf[i] = 0.f;
        }
        OP_REQUIRES(ctx, rc == 0, errors::Internal("bts_lpg_bwd failed with code ", rc));
    }
};

REGISTER_KERNEL_BUILDER(Name("LocalPlanarGuidance").Device(DEVICE_CPU), LpgOp<false>);
REGISTER_KERNEL_BUILDER(Name("LocalPlanarGuidanceGrad").Device(DEVICE_CPU), LpgGradOp<false>);
#if GOOGLE_CUDA
REGISTER_KERNEL_BUILDER(Name("LocalPlanarGuidance").Device(DEVICE_GPU), LpgOp<true>);
REGISTER_KERNEL_BUILDER(Name("LocalPlanarGuidanceGrad").Device(DEVICE_GPU), LpgGradOp<true>);
#endif

}  // namespace bts_b200_tf
