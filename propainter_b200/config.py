"""Execution switches (module-level; read at call time).

LINEAR_TF32     plain Linear layers of the transformer (q/k/v, proj, fc1, fc2 = 807 GFLOP per generator call)
                run as TF32 tensor-core GEMMs (fp32 accumulate) instead of cuBLAS' fp32 SIMT sgemm.  Same
                precision class as the reference's own CUDA convs (cuDNN TF32 is torch's default) and as our
                attention / deform-align kernels.  Set False for fp32-exact library GEMMs (tests do, to
                isolate kernel error).
CUDNN_BENCHMARK let cuDNN autotune conv algorithms during graph warm-up.
CUDA_GRAPHS     replay each stage as a captured CUDA graph per shape signature (propainter_b200/graphs.py).
FUSED_EPILOGUE  conv bias + activation through pp_bias_act (one pass) instead of cuDNN's bias add_ + ATen activation.
UMMA_CONV       the convolutions of the two recurrent propagation scans (offset nets, backbones, deformable-conv GEMM) run on
                the wgmma implicit-GEMM kernel pp_conv2d_umma (TF32 products, fused bias / activation / residual / concat
                epilogue) instead of cuDNN + pp_bias_act + the mma.sync deform kernel.  True / False force one plan;
                "hybrid" keeps the library convs and replaces only the deformable conv by pp_deform_gather + a 1x1
                pp_conv2d_umma GEMM; "hoisted" additionally convolves the step-independent input channels of
                conv_offset.0 / backbone.0 once per scan (library convs, pp_bias_act_pre); "auto" (default) times the plans of a scan once per shape during graph warm-up
                (autotune.pick) and replays the fastest.  Environment: PP_UMMA_CONV=1|0|hybrid|hoisted|auto.
SCAN_PRIORITY   capture the recurrent propagation scans as high-priority branches of their stage graphs (graphs.high_priority).
                Environment: PP_SCAN_PRIORITY=0|1.
GRAPH_MAX_INPUT_BYTES  stage calls whose inputs exceed this run eagerly instead of as a captured graph (memory: a capture keeps
                its whole working set alive in a private pool).
HALF_OPERANDS   RAFT's refinement-loop convs (convc1, convc2, convf2, the motion conv, the four SepConvGRU gate convs,
                flow_head.conv1) take fp16 operands with fp32 accumulation, on the all-pairs correlation plan.  fp16 has TF32's
                10 mantissa bits, so this replaces TF32 by the same precision class at twice the tensor rate and half the bytes;
                it is active only while cuDNN may use TF32 (torch.backends.cudnn.allow_tf32), so a strict-fp32 run stays
                strict.  The recurrent state, the coordinates and every other conv stay fp32 (DESIGN.md §4 "Precision").
                The generator's transformer takes fp16 operands the same way: every LayerNorm writes its output as fp16,
                the fused QKV, pooled K/V, proj, fc1 and fc2 Linear layers run on fp16 weights and biases with fp32
                accumulation and fp32 split-K reductions and write fp16, the depthwise pooling, the window attention (f16
                wgmma / mma.sync kernels, fp32 softmax and accumulators) and the fold / unfold read and write fp16 rows while
                computing in fp32, and each sublayer's fp16 output enters the fp32 residual stream in the next LayerNorm.
                This is active only while those Linear layers would run TF32 anyway (LINEAR_TF32 or
                torch.backends.cuda.matmul.allow_tf32, CUDA tensors), so a strict-fp32 run stays strict.
                Where cuDNN may use TF32 (half_convs) it also runs the per-step convs of the two recurrent propagation
                scans (plan 0 of UMMA_CONV) on the fp16 instance of pp_conv2d_umma; their states stay fp32.
                There it also runs two clip encoders on fp16 operands: the generator's frame encoder (fp16 input, weights
                and maps, the grouped layers' inputs written into their group slots by the previous epilogue) and RAFT's
                context encoder cnet (pp_bias_act epilogues with an fp16 residual); both widen their last conv's output
                to fp32, so the encoder features, `net` and `inp` stay fp32.  RAFT's feature encoder fnet stays TF32.
                Environment: PP_HALF_OPERANDS=0|1.
AUTOTUNE        time numerically equivalent plans of a step once per shape during warm-up and keep the faster
                (propainter_b200/autotune.py): grouped conv vs per-group dense convs, conv + pp_bias_act vs cuDNN's fused
                conv-bias-ReLU.
"""
import contextlib
import os

import torch

LINEAR_TF32 = True
CUDNN_BENCHMARK = True
CUDA_GRAPHS = True
FUSED_EPILOGUE = True
AUTOTUNE = True
GRAPH_MAX_INPUT_BYTES = 256 << 20      # C2 calls (<= ~170 MB) are graphed; 720p calls run eagerly (80 GB)
SCAN_PRIORITY = os.environ.get("PP_SCAN_PRIORITY", "1") != "0"
HALF_OPERANDS = os.environ.get("PP_HALF_OPERANDS", "1") != "0"
_u = os.environ.get("PP_UMMA_CONV", "auto")
UMMA_CONV = _u if _u in ("auto", "hybrid", "hoisted") else (_u != "0")


def half_convs():
    """whether RAFT's refinement-loop convs run on fp16 operands now (HALF_OPERANDS where cuDNN may use TF32)"""
    return bool(HALF_OPERANDS) and torch.backends.cudnn.allow_tf32


def half_linears():
    """whether the transformer runs on fp16 operands now (HALF_OPERANDS where its Linear layers would run TF32)"""
    return bool(HALF_OPERANDS) and (bool(LINEAR_TF32) or torch.backends.cuda.matmul.allow_tf32)


@contextlib.contextmanager
def fp32_reductions():
    """fp16 cuBLAS GEMMs with their split-K partial sums reduced in fp32 (else cuBLAS may reduce them in fp16)"""
    prev = torch.backends.cuda.matmul.allow_fp16_reduced_precision_reduction
    torch.backends.cuda.matmul.allow_fp16_reduced_precision_reduction = False
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_fp16_reduced_precision_reduction = prev


@contextlib.contextmanager
def linear_precision():
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = bool(LINEAR_TF32) or prev
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev


@contextlib.contextmanager
def cudnn_autotune():
    prev = torch.backends.cudnn.benchmark
    torch.backends.cudnn.benchmark = bool(CUDNN_BENCHMARK) or prev
    try:
        yield
    finally:
        torch.backends.cudnn.benchmark = prev
