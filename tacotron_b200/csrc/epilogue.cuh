// epilogue.cuh -- the fused epilogue shared by the SIMT and tensor-core (wgmma) contraction kernels.
// epi(v) = (act(v + bias[n]) * scale[n] + shift[n]) * keep[row][n]*keep_scale + residual[row][n]
// (tf.layers.dense/conv1d bias+activation, inference-mode batch_normalization affine,
//  tf.layers.dropout with an explicit keep mask, CBHG residual: models/ops.py:54-92,
//  models/tacotron.py:38-44)
#pragma once
#include "common.cuh"

struct EpiParams {
    float*         Y;
    int64_t        ldy;
    const float*   bias;
    const float*   scale;
    const float*   shift;
    const uint8_t* keep;
    const float*   residual;
    int64_t        ldr;
    const float*   hx;
    int64_t        ldhx;
    float          keep_scale;
    int            act;
    int            N;       // valid output columns (for keep-mask row stride and bounds)
    const float*   bias_utt; // [B][ldbu] per-utterance bias or NULL (row / T = utterance)
    int64_t        ldbu;
    int            T;
};

__device__ __forceinline__ float epi_value(const EpiParams& e, int64_t row, int col, float v) {
    if (e.bias_utt) {
        const float bu = __ldg(e.bias_utt + (row / e.T) * e.ldbu + col);
        v += e.bias ? __ldg(e.bias + col) + bu : bu;
    } else if (e.bias) {
        v += __ldg(e.bias + col);
    }
    v = apply_act(v, e.act);
    if (e.scale) v = v * __ldg(e.scale + col);
    if (e.shift) v = v + __ldg(e.shift + col);
    if (e.keep) v = e.keep[row * (int64_t)e.N + col] ? v * e.keep_scale : 0.0f;
    if (e.residual) v += e.residual[row * e.ldr + col];
    return v;
}

// highway combine (models/ops.py:32-45): H = relu(h + bH), T = sigmoid(t + bT), out = H*T + x*(1-T)
// bias holds [bH | bT] (2U entries); col in [0,U)
__device__ __forceinline__ float epi_highway(const EpiParams& e, int64_t row, int col, int U, float h, float t) {
    if (e.bias) { h += __ldg(e.bias + col); t += __ldg(e.bias + U + col); }
    float H = fmaxf(h, 0.0f);
    float T = sigmoidf_acc(t);
    float x = e.hx[row * e.ldhx + col];
    return H * T + x * (1.0f - T);
}
