// host_mel_tables.h — host-side tables of the mel kernel (twiddles, sparse Slaney filterbank).
// Part of the single translation unit w2l_api.cu (included there, in this order).
#pragma once

// ------------------------------------------------------------------------------------------------
// mel tables (host, double precision) — librosa 0.7.0 filters.mel(16000, 800, 80, 55, 7600), Slaney
// ------------------------------------------------------------------------------------------------
static double hz_to_mel(double f) {
    const double f_sp = 200.0 / 3.0, min_log_hz = 1000.0, min_log_mel = min_log_hz / f_sp, logstep = std::log(6.4) / 27.0;
    return f >= min_log_hz ? min_log_mel + std::log(f / min_log_hz) / logstep : f / f_sp;
}
static double mel_to_hz(double m) {
    const double f_sp = 200.0 / 3.0, min_log_hz = 1000.0, min_log_mel = min_log_hz / f_sp, logstep = std::log(6.4) / 27.0;
    return m >= min_log_mel ? min_log_hz * std::exp(logstep * (m - min_log_mel)) : f_sp * m;
}
static void build_mel_basis(std::vector<float>* dense) {
    const int nm = MEL_BANDS, nb = MEL_BINS;
    dense->assign((size_t)nm * nb, 0.0f);
    std::vector<double> mel_f(nm + 2);
    const double m0 = hz_to_mel(55.0), m1 = hz_to_mel(7600.0);
    const double step = (m1 - m0) / (nm + 1);
    for (int i = 0; i < nm + 2; ++i) mel_f[i] = mel_to_hz(i == nm + 1 ? m1 : m0 + i * step);
    for (int i = 0; i < nm; ++i) {
        const double fd0 = mel_f[i + 1] - mel_f[i], fd1 = mel_f[i + 2] - mel_f[i + 1];
        const double enorm = 2.0 / (mel_f[i + 2] - mel_f[i]);
        for (int k = 0; k < nb; ++k) {
            const double f = 8000.0 * k / (nb - 1);
            const double lower = -(mel_f[i] - f) / fd0, upper = (mel_f[i + 2] - f) / fd1;
            const float w32 = (float)std::max(0.0, std::min(lower, upper));
            (*dense)[(size_t)i * nb + k] = (float)((double)w32 * enorm);
        }
    }
}

static int init_mel_tables(w2l_ctx* ctx) {
    std::vector<double2> tw(MEL_BINS);  // exp(-2 pi i m / 800), m = 0..400
    const long double kTwoPi = 2.0L * 3.141592653589793238462643383279502884L;
    for (int m = 0; m < MEL_BINS; ++m) {
        const long double a = -kTwoPi * m / MEL_NFFT;
        tw[m] = make_double2((double)cosl(a), (double)sinl(a));
    }
    std::vector<float> dense;
    build_mel_basis(&dense);
    std::vector<float> vals;
    std::vector<int> off(MEL_BANDS), start(MEL_BANDS), len(MEL_BANDS);
    for (int i = 0; i < MEL_BANDS; ++i) {
        int a = -1, b = -1;
        for (int k = 0; k < MEL_BINS; ++k)
            if (dense[(size_t)i * MEL_BINS + k] != 0.0f) { if (a < 0) a = k; b = k; }
        off[i] = (int)vals.size();
        start[i] = a < 0 ? 0 : a;
        len[i] = a < 0 ? 0 : b - a + 1;
        for (int k = 0; k < len[i]; ++k) vals.push_back(dense[(size_t)i * MEL_BINS + start[i] + k]);
    }
    CKR(ctx->mel_tw.grow(ctx, tw.size() * sizeof(double2)));
    CKR(ctx->mel_bvals.grow(ctx, vals.size() * 4));
    CKR(ctx->mel_boff.grow(ctx, MEL_BANDS * 4));
    CKR(ctx->mel_bstart.grow(ctx, MEL_BANDS * 4));
    CKR(ctx->mel_blen.grow(ctx, MEL_BANDS * 4));
    CK(cudaMemcpy(ctx->mel_tw, tw.data(), tw.size() * sizeof(double2), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(ctx->mel_bvals, vals.data(), vals.size() * 4, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(ctx->mel_boff, off.data(), MEL_BANDS * 4, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(ctx->mel_bstart, start.data(), MEL_BANDS * 4, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(ctx->mel_blen, len.data(), MEL_BANDS * 4, cudaMemcpyHostToDevice));
    CK(cudaFuncSetAttribute(mel_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMelSmemBytes));
    CK(cudaFuncSetAttribute(mel_ring_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMelSmemBytes));
    return W2L_OK;
}
