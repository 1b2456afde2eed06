// netspec.h — the three networks of the hot path as data (host only, no CUDA).
//
// These tables are the product's statement of the architectures defined by
//   /root/reference/models/wav2lip.py:12-85   (Wav2Lip generator)
//   /root/reference/models/wav2lip.py:131-152 (Wav2Lip_disc_qual)
//   /root/reference/models/syncnet.py:11-53   (SyncNet_color)
// with the reference's module paths as names, so that the Python mirror can build nn.Modules with
// identical state_dict keys from them (w2l_net_layer_info) and the planner can wire the kernels.
// They are generated from per-stage descriptors rather than listed layer by layer.
#pragma once

#include <string>
#include <vector>

#include "../../include/w2l.h"

namespace w2l {

struct Layer {
    std::string name;
    int kind;
    int cin, cout, kh, kw, sh, sw, ph, pw, out_pad;
    bool residual;
    bool bare_keys = false;   // parameters are "<name>.weight" / "<name>.bias" (plain nn.Conv2d members: S3FD) instead of "<name>.conv_block.0.*"
    int cout_real = 0;        // > 0: the tensor has this many output channels, `cout` is its 16-padded width (S3FD heads: 2 / 4)
};

inline Layer mk(const std::string& name, int kind, int cin, int cout, int k, int sh, int sw, int p, int op = 0,
                bool res = false) {
    return Layer{name, kind, cin, cout, k, k, sh, sw, p, p, op, res};
}

// A down-sampling stage: one strided conv followed by `nres` residual 3x3 convs at the new width.
inline void add_stage(std::vector<Layer>& L, const std::string& prefix, int first_idx, bool nested, int kind, int cin,
                      int cout, int k, int sh, int sw, int p, int nres, int kres = 3) {
    auto nm = [&](int j) {
        return nested ? prefix + "." + std::to_string(j) : prefix + "." + std::to_string(first_idx + j);
    };
    L.push_back(mk(nm(0), kind, cin, cout, k, sh, sw, p));
    for (int j = 1; j <= nres; ++j) L.push_back(mk(nm(j), kind, cout, cout, kres, 1, 1, kres / 2, 0, kind == W2L_BLOCK_CONV_BN_RELU));
}

// The mel encoder shared (up to one block) by the generator and SyncNet:
// 80x16 -> (3,1) -> 27x16 -> (3,3) -> 9x6 -> (3,2) -> 3x3 -> 1x1.   n256 = residual blocks at 256 channels.
inline void add_audio_encoder(std::vector<Layer>& L, int n256) {
    const std::string pre = "audio_encoder";
    int idx = 0;
    add_stage(L, pre, idx, false, W2L_BLOCK_CONV_BN_RELU, 1, 32, 3, 1, 1, 1, 2); idx += 3;
    add_stage(L, pre, idx, false, W2L_BLOCK_CONV_BN_RELU, 32, 64, 3, 3, 1, 1, 2); idx += 3;
    add_stage(L, pre, idx, false, W2L_BLOCK_CONV_BN_RELU, 64, 128, 3, 3, 3, 1, 2); idx += 3;
    add_stage(L, pre, idx, false, W2L_BLOCK_CONV_BN_RELU, 128, 256, 3, 3, 2, 1, n256); idx += 1 + n256;
    L.push_back(mk(pre + "." + std::to_string(idx++), W2L_BLOCK_CONV_BN_RELU, 256, 512, 3, 1, 1, 0));
    L.push_back(mk(pre + "." + std::to_string(idx++), W2L_BLOCK_CONV_BN_RELU, 512, 512, 1, 1, 1, 0));
}

struct GeneratorSpec {
    std::vector<Layer> layers;
    // index ranges into `layers`
    std::vector<std::vector<int>> face_enc;  // 7 stages
    std::vector<int> audio_enc;              // 13 blocks
    std::vector<std::vector<int>> face_dec;  // 7 stages
    int output_block0;
    // skip concatenation (wav2lip.py:108): decoder stage k's output (dec_c[k] channels) is concatenated with the encoder
    // feature of the same resolution hw[k] (skip_c[k] channels); stage k + 1 reads both
    int hw[7] = {1, 3, 6, 12, 24, 48, 96};
    int dec_c[7] = {512, 512, 512, 384, 256, 128, 64};
    int skip_c[7] = {512, 512, 256, 128, 64, 32, 16};
};

inline GeneratorSpec build_generator_spec() {
    GeneratorSpec g;
    auto& L = g.layers;
    const int C = W2L_BLOCK_CONV_BN_RELU, T = W2L_BLOCK_CONVT_BN_RELU;
    // face encoder: 96 -> 48 -> 24 -> 12 -> 6 -> 3 -> 1
    const int enc_c[6] = {16, 32, 64, 128, 256, 512};
    const int enc_res[6] = {0, 2, 3, 2, 2, 1};
    int cin = 6;
    for (int i = 0; i < 6; ++i) {
        const size_t b = L.size();
        const std::string pre = "face_encoder_blocks." + std::to_string(i);
        if (i == 0) add_stage(L, pre, 0, true, C, cin, enc_c[i], 7, 1, 1, 3, 0);
        else add_stage(L, pre, 0, true, C, cin, enc_c[i], 3, 2, 2, 1, enc_res[i]);
        std::vector<int> idx;
        for (size_t k = b; k < L.size(); ++k) idx.push_back((int)k);
        g.face_enc.push_back(idx);
        cin = enc_c[i];
    }
    {
        const size_t b = L.size();
        L.push_back(mk("face_encoder_blocks.6.0", C, 512, 512, 3, 1, 1, 0));
        L.push_back(mk("face_encoder_blocks.6.1", C, 512, 512, 1, 1, 1, 0));
        g.face_enc.push_back({(int)b, (int)b + 1});
    }
    {
        const size_t b = L.size();
        add_audio_encoder(L, 1);
        for (size_t k = b; k < L.size(); ++k) g.audio_enc.push_back((int)k);
    }
    // decoder: input width of stage k = (own output of stage k-1) + (encoder skip of the same resolution)
    const int *dec_c = g.dec_c, *skip_c = g.skip_c;
    const int dec_res[7] = {0, 1, 2, 2, 2, 2, 2};
    {
        const size_t b = L.size();
        L.push_back(mk("face_decoder_blocks.0.0", C, 512, 512, 1, 1, 1, 0));
        g.face_dec.push_back({(int)b});
    }
    for (int k = 1; k < 7; ++k) {
        const size_t b = L.size();
        const std::string pre = "face_decoder_blocks." + std::to_string(k);
        const int in_c = dec_c[k - 1] + skip_c[k - 1];
        if (k == 1) L.push_back(mk(pre + ".0", T, in_c, dec_c[k], 3, 1, 1, 0, 0));      // 1x1 -> 3x3
        else L.push_back(mk(pre + ".0", T, in_c, dec_c[k], 3, 2, 2, 1, 1));              // H -> 2H
        for (int j = 1; j <= dec_res[k]; ++j) L.push_back(mk(pre + "." + std::to_string(j), C, dec_c[k], dec_c[k], 3, 1, 1, 1, 0, true));
        std::vector<int> idx;
        for (size_t q = b; q < L.size(); ++q) idx.push_back((int)q);
        g.face_dec.push_back(idx);
    }
    g.output_block0 = (int)L.size();
    L.push_back(mk("output_block.0", C, dec_c[6] + skip_c[6], 32, 3, 1, 1, 1));
    return g;
}

struct SyncnetSpec {
    std::vector<Layer> layers;
    std::vector<int> face_enc, audio_enc;
};

inline SyncnetSpec build_syncnet_spec() {
    SyncnetSpec s;
    auto& L = s.layers;
    const int C = W2L_BLOCK_CONV_BN_RELU;
    const std::string pre = "face_encoder";
    int idx = 0;
    L.push_back(mk(pre + ".0", C, 15, 32, 7, 1, 1, 3)); idx = 1;
    // 48x96 -> k5 s(1,2) p1 -> 46x47
    L.push_back(mk(pre + ".1", C, 32, 64, 5, 1, 2, 1));
    L.push_back(mk(pre + ".2", C, 64, 64, 3, 1, 1, 1, 0, true));
    L.push_back(mk(pre + ".3", C, 64, 64, 3, 1, 1, 1, 0, true));
    idx = 4;
    add_stage(L, pre, idx, false, C, 64, 128, 3, 2, 2, 1, 3); idx += 4;
    add_stage(L, pre, idx, false, C, 128, 256, 3, 2, 2, 1, 2); idx += 3;
    add_stage(L, pre, idx, false, C, 256, 512, 3, 2, 2, 1, 2); idx += 3;
    L.push_back(mk(pre + "." + std::to_string(idx++), C, 512, 512, 3, 2, 2, 1));
    L.push_back(mk(pre + "." + std::to_string(idx++), C, 512, 512, 3, 1, 1, 0));
    L.push_back(mk(pre + "." + std::to_string(idx++), C, 512, 512, 1, 1, 1, 0));
    for (size_t k = 0; k < L.size(); ++k) s.face_enc.push_back((int)k);
    const size_t b = L.size();
    add_audio_encoder(L, 2);
    for (size_t k = b; k < L.size(); ++k) s.audio_enc.push_back((int)k);
    return s;
}

struct DiscSpec {
    std::vector<Layer> layers;  // 13 nonorm blocks; binary_pred (512->1, sigmoid) is handled by the head kernel
};

inline DiscSpec build_disc_spec() {
    DiscSpec d;
    auto& L = d.layers;
    const int NN = W2L_BLOCK_CONV_LRELU;
    const std::string pre = "face_encoder_blocks.";
    L.push_back(mk(pre + "0.0", NN, 3, 32, 7, 1, 1, 3));
    // 48x96 -> 48x48 -> 24 -> 12 (5x5 kernels) -> 6 -> 3 (3x3) -> 1
    L.push_back(mk(pre + "1.0", NN, 32, 64, 5, 1, 2, 2));
    L.push_back(mk(pre + "1.1", NN, 64, 64, 5, 1, 1, 2));
    const int c[5] = {64, 128, 256, 512, 512};
    for (int i = 2; i <= 5; ++i) {
        const int k = (i <= 3) ? 5 : 3;
        const std::string p2 = pre + std::to_string(i);
        L.push_back(mk(p2 + ".0", NN, c[i - 2], c[i - 1], k, 2, 2, k / 2));
        L.push_back(mk(p2 + ".1", NN, c[i - 1], c[i - 1], k, 1, 1, k / 2));
    }
    L.push_back(mk(pre + "6.0", NN, 512, 512, 3, 1, 1, 0));
    L.push_back(mk(pre + "6.1", NN, 512, 512, 1, 1, 1, 0));
    return d;
}

// face_detection/detection/sfd/net_s3fd.py:22-129.  Backbone layers 0..18 (conv + ReLU), heads 19..30 (conv only, output
// channels padded to 16).  Pools, L2Norm and the taps are wired by the planner (host_plans.cuh: build_s3fd_plan).
struct S3fdSpec {
    std::vector<Layer> layers;
};

inline S3fdSpec build_s3fd_spec() {
    S3fdSpec s;
    auto& L = s.layers;
    const int R = W2L_BLOCK_CONV_RELU, P = W2L_BLOCK_CONV_PLAIN;
    auto add = [&](const char* name, int kind, int cin, int cout, int k, int stride, int pad, int cout_real = 0) {
        Layer l = mk(name, kind, cin, cout, k, stride, stride, pad);
        l.bare_keys = true;
        l.cout_real = cout_real;
        L.push_back(l);
    };
    add("conv1_1", R, 3, 64, 3, 1, 1);    add("conv1_2", R, 64, 64, 3, 1, 1);
    add("conv2_1", R, 64, 128, 3, 1, 1);  add("conv2_2", R, 128, 128, 3, 1, 1);
    add("conv3_1", R, 128, 256, 3, 1, 1); add("conv3_2", R, 256, 256, 3, 1, 1); add("conv3_3", R, 256, 256, 3, 1, 1);
    add("conv4_1", R, 256, 512, 3, 1, 1); add("conv4_2", R, 512, 512, 3, 1, 1); add("conv4_3", R, 512, 512, 3, 1, 1);
    add("conv5_1", R, 512, 512, 3, 1, 1); add("conv5_2", R, 512, 512, 3, 1, 1); add("conv5_3", R, 512, 512, 3, 1, 1);
    add("fc6", R, 512, 1024, 3, 1, 3);    add("fc7", R, 1024, 1024, 1, 1, 0);
    add("conv6_1", R, 1024, 256, 1, 1, 0); add("conv6_2", R, 256, 512, 3, 2, 1);
    add("conv7_1", R, 512, 128, 1, 1, 0);  add("conv7_2", R, 128, 256, 3, 2, 1);
    const char* taps[6] = {"conv3_3_norm", "conv4_3_norm", "conv5_3_norm", "fc7", "conv6_2", "conv7_2"};
    const int tap_c[6] = {256, 512, 512, 1024, 512, 256};
    for (int i = 0; i < 6; ++i) {
        add((std::string(taps[i]) + "_mbox_conf").c_str(), P, tap_c[i], 16, 3, 1, 1, i == 0 ? 4 : 2);
        add((std::string(taps[i]) + "_mbox_loc").c_str(), P, tap_c[i], 16, 3, 1, 1, 4);
    }
    return s;
}

}  // namespace w2l
