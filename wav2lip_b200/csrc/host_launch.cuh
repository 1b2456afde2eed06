// host_launch.cuh — kernel instantiation tables and the one function that launches a conv Op (generic / patch /
// fused transposed-conv kernel), with the per-device shared-memory attribute and the PDL launch attribute.
// Part of the single translation unit w2l_api.cu (included there, in this order).
#pragma once

// ------------------------------------------------------------------------------------------------
// conv kernel dispatch
// ------------------------------------------------------------------------------------------------
typedef void (*ConvKernelFn)(const ConvParams);
// cm: the channel-major form of the (BN, BK, MT = 1) instantiation (conv_igemm.cuh, kCM)
struct ConvKernelEntry { int BN, BK; bool bf16, head; ConvKernelFn fn; int smem; uint64_t attr_set; int mt; int threads; bool cm; };

#define W2L_CONV_ENTRY(BN_, BK_)                                                                                                        \
    {BN_, BK_, false, false, conv_igemm_kernel<BN_, BK_, false, false>, ConvCfg<BN_, BK_>::kSmemBytes, 0, 1, ConvCfg<BN_, BK_>::kThreads, false}, \
    {BN_, BK_, true, false, conv_igemm_kernel<BN_, BK_, true, false>, ConvCfg<BN_, BK_>::kSmemBytes, 0, 1, ConvCfg<BN_, BK_>::kThreads, false}
#define W2L_CONV_ENTRY_MT2(BN_, BK_)                                                                                                    \
    {BN_, BK_, false, false, conv_igemm_kernel<BN_, BK_, false, false, 2>, ConvCfg<BN_, BK_, 2>::kSmemBytes, 0, 2, ConvCfg<BN_, BK_, 2>::kThreads, false}, \
    {BN_, BK_, true, false, conv_igemm_kernel<BN_, BK_, true, false, 2>, ConvCfg<BN_, BK_, 2>::kSmemBytes, 0, 2, ConvCfg<BN_, BK_, 2>::kThreads, false}
#define W2L_CONV_ENTRY_CM(BN_, BK_)                                                                                                     \
    {BN_, BK_, false, false, conv_igemm_kernel<BN_, BK_, false, false, 1, true>, ConvCfg<BN_, BK_, 1, true>::kSmemBytes, 0, 1, ConvCfg<BN_, BK_, 1, true>::kThreads, true}, \
    {BN_, BK_, true, false, conv_igemm_kernel<BN_, BK_, true, false, 1, true>, ConvCfg<BN_, BK_, 1, true>::kSmemBytes, 0, 1, ConvCfg<BN_, BK_, 1, true>::kThreads, true}

static ConvKernelEntry g_conv_kernels[] = {
    W2L_CONV_ENTRY(16, 16), W2L_CONV_ENTRY(16, 32), W2L_CONV_ENTRY(16, 64),
    W2L_CONV_ENTRY(32, 16), W2L_CONV_ENTRY(32, 32), W2L_CONV_ENTRY(32, 64),
    W2L_CONV_ENTRY(64, 16), W2L_CONV_ENTRY(64, 32), W2L_CONV_ENTRY(64, 64),
    W2L_CONV_ENTRY(128, 16), W2L_CONV_ENTRY(128, 32), W2L_CONV_ENTRY(128, 64),
    W2L_CONV_ENTRY_MT2(64, 64), W2L_CONV_ENTRY_MT2(64, 32),
    W2L_CONV_ENTRY_CM(128, 64),
    {32, 16, false, true, conv_igemm_kernel<32, 16, false, true>, ConvCfg<32, 16>::kSmemBytes, 0, 1, ConvCfg<32, 16>::kThreads, false},
    {32, 16, true, true, conv_igemm_kernel<32, 16, true, true>, ConvCfg<32, 16>::kSmemBytes, 0, 1, ConvCfg<32, 16>::kThreads, false},
};

static ConvKernelEntry* find_conv_kernel(int BN, int BK, bool bf16, bool head, int mt = 1, bool cm = false) {
    for (auto& e : g_conv_kernels)
        if (e.BN == BN && e.BK == BK && e.bf16 == bf16 && e.head == head && e.mt == mt && e.cm == cm) return &e;
    return nullptr;
}

typedef void (*PatchKernelFn)(const PatchParams);
struct PatchKernelEntry { int BN, BK; bool bf16, head; PatchKernelFn fn; uint64_t attr_set; };
#define W2L_PATCH_ENTRY(BN_, BK_)                                                    \
    {BN_, BK_, false, false, conv_patch_kernel<BN_, BK_, false, false>, 0},    \
    {BN_, BK_, true, false, conv_patch_kernel<BN_, BK_, true, false>, 0}
static PatchKernelEntry g_patch_kernels[] = {
    W2L_PATCH_ENTRY(16, 16), W2L_PATCH_ENTRY(16, 32), W2L_PATCH_ENTRY(16, 64),
    W2L_PATCH_ENTRY(32, 16), W2L_PATCH_ENTRY(32, 32), W2L_PATCH_ENTRY(32, 64),
    W2L_PATCH_ENTRY(64, 16), W2L_PATCH_ENTRY(64, 32), W2L_PATCH_ENTRY(64, 64),
    {32, 16, false, true, conv_patch_kernel<32, 16, false, true>, 0},
    {32, 16, true, true, conv_patch_kernel<32, 16, true, true>, 0},
};
static PatchKernelEntry* find_patch_kernel(int BN, int BK, bool bf16, bool head) {
    for (auto& e : g_patch_kernels)
        if (e.BN == BN && e.BK == BK && e.bf16 == bf16 && e.head == head) return &e;
    return nullptr;
}

typedef void (*CtKernelFn)(const ConvTParams);
struct CtKernelEntry { int BK; bool bf16; CtKernelFn fn; uint64_t attr_set; };
static CtKernelEntry g_ct_kernels[] = {
    {32, false, convt_fused_kernel<32, false>, 0}, {32, true, convt_fused_kernel<32, true>, 0},
};
constexpr int kCtSmemMax = 227 * 1024;

// cudaFuncAttributeMaxDynamicSharedMemorySize is a per-device property of a kernel: remember it per device (one bit
// each), so that contexts on several GPUs of one process all get it
static int ensure_smem_attr(uint64_t* mask, int device, const void* fn, int bytes) {
    const uint64_t bit = 1ull << (device & 63);
    if (*mask & bit) return W2L_OK;
    CK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    *mask |= bit;
    return W2L_OK;
}

// One launch, optionally with programmatic stream serialization (the kernels call griddepcontrol.wait before they
// touch global memory, so their prologue overlaps the previous kernel's tail).
template <typename P>
static cudaError_t launch_k(void (*fn)(const P), int grid, int block, size_t smem, cudaStream_t st, const P& p, bool pdl) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3((unsigned)grid, 1, 1);
    cfg.blockDim = dim3((unsigned)block, 1, 1);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = pdl ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, fn, p);
}

// the w2l_kernel_info row of one conv Op (test aid: which kernel instantiation the launch uses)
static void op_kernel_info(const w2l_ctx* ctx, const Op& op, w2l_kernel_info* k) {
    memset(k, 0, sizeof(*k));
    snprintf(k->name, sizeof(k->name), "%s", op.name.c_str());
    k->family = op.ctf ? W2L_KFAM_CONVT_FUSED : op.patch ? W2L_KFAM_PATCH : W2L_KFAM_IGEMM;
    k->bn = op.BN; k->bk = op.BK; k->mt = op.MT; k->head = op.head ? 1 : 0;
    k->bf16 = ctx->bf16 ? 1 : 0; k->x2 = ctx->x2 ? 1 : 0;
    k->tma_epi = (!op.ctf && !op.patch && op.cp.tma_epi) ? 1 : 0;
    k->fold = op.fold ? 1 : 0;
    k->m_tiles = op.m_tiles; k->n_tiles = op.n_tiles; k->grid = op.grid;
    // the box of output pixels one M tile covers (width x height x images)
    if (op.ctf) { k->box_w = 8; k->box_h = 16; k->box_n = 1; }
    else if (op.patch) { k->box_w = kPatchTileW; k->box_h = op.patch_th; k->box_n = 1; k->patch_th = op.patch_th; }
    else { k->box_w = op.cp.bw; k->box_h = op.cp.bh; k->box_n = op.cp.bn; }
}

static int launch_conv(w2l_ctx* ctx, const Op& op, cudaStream_t st, bool pdl = true) {
    pdl = pdl && ctx->use_pdl;
    if (op.ctf) {
        CtKernelEntry* e = nullptr;
        for (auto& k : g_ct_kernels) if (k.BK == op.BK && k.bf16 == ctx->bf16) e = &k;
        if (!e) return fail(W2L_EINVAL, "no fused convT kernel for BK=%d", op.BK);
        CKR(ensure_smem_attr(&e->attr_set, ctx->device, (const void*)e->fn, kCtSmemMax));
        CK(launch_k(e->fn, op.grid, kCtThreads, op.dyn_smem, st, op.tp, pdl));
        ctx->launches++;
        return W2L_OK;
    }
    if (op.patch) {
        PatchKernelEntry* e = find_patch_kernel(op.BN, op.BK, ctx->bf16, op.head);
        if (!e) return fail(W2L_EINVAL, "no patch kernel for BN=%d BK=%d head=%d", op.BN, op.BK, (int)op.head);
        CKR(ensure_smem_attr(&e->attr_set, ctx->device, (const void*)e->fn, kSmemMax));
        CK(launch_k(e->fn, op.grid, kPatchThreads, op.dyn_smem, st, op.pp, pdl));
        ctx->launches++;
        return W2L_OK;
    }
    ConvKernelEntry* e = find_conv_kernel(op.BN, op.BK, ctx->bf16, op.head, op.MT, op.cm);
    if (!e) return fail(W2L_EINVAL, "no conv kernel for BN=%d BK=%d head=%d MT=%d cm=%d", op.BN, op.BK, (int)op.head, op.MT, (int)op.cm);
    CKR(ensure_smem_attr(&e->attr_set, ctx->device, (const void*)e->fn, e->smem));
    CK(launch_k(e->fn, op.grid, e->threads, (size_t)e->smem, st, op.cp, pdl));
    ctx->launches++;
    return W2L_OK;
}
