// unet_engine.cu - the UNetSeeInDark training / inference step as a fixed launch sequence over the
// wgmma tiles (unet_prims.cu) and the HBM-bound helpers (unet_ew.cu).
//
// Reference: models/arch/Unet.py:48-91 (forward), models/ELD_model.py:411-420,469-475 (L1 loss,
// backward, Adam).  Activations NHWC bf16; torch.cat (Unet.py:69,74,79,84) is free: the deconv and
// the encoder conv write disjoint channel ranges of one "cat" buffer.  Parameters and gradients are
// flat fp32 buffers in state_dict order (so released checkpoints map 1:1 and DDP all-reduces one buffer).
#include "common.cuh"
#include "unet_prims.h"
#include "unet_ew.h"
#include <cuda_bf16.h>
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>
#include <new>

namespace eld {

enum { L_CONV3 = 0, L_DECONV = 1, L_CONV1 = 2 };
enum { I_C11 = 0, I_C12, I_C21, I_C22, I_C31, I_C32, I_C41, I_C42, I_C51, I_C52, I_UP6, I_C61, I_C62, I_UP7,
       I_C71, I_C72, I_UP8, I_C81, I_C82, I_UP9, I_C91, I_C92, I_C10 };
struct LayerSpec { const char* name; int type, cin, cout, lvl, src, skip; };
struct Layer : LayerSpec { size_t w_off, b_off, wf_off, wd_off; };

// UNetSeeInDark (Unet.py:11-46) in state_dict order, which is a topological order of its forward graph.  lvl: the grid of
// the layer's output, 1/2^lvl of the frame (a deconv's is the fine grid it writes).  src: the layer whose output it reads
// (-1 = the input frame x; a pool between two encoder levels does not change who produced the tensor).  skip: for the four
// concatenating convs, the encoder layer behind the skip half of their input (Unet.py:69,74,79,84).  Every buffer, launch
// and backward step of the engine is derived from this table.
static const LayerSpec kLayers[] = {
    //  name       type      cin  cout lvl  src    skip
    { "conv1_1",  L_CONV3,    4,  32, 0, -1,    -1 },
    { "conv1_2",  L_CONV3,   32,  32, 0, I_C11, -1 },
    { "conv2_1",  L_CONV3,   32,  64, 1, I_C12, -1 },
    { "conv2_2",  L_CONV3,   64,  64, 1, I_C21, -1 },
    { "conv3_1",  L_CONV3,   64, 128, 2, I_C22, -1 },
    { "conv3_2",  L_CONV3,  128, 128, 2, I_C31, -1 },
    { "conv4_1",  L_CONV3,  128, 256, 3, I_C32, -1 },
    { "conv4_2",  L_CONV3,  256, 256, 3, I_C41, -1 },
    { "conv5_1",  L_CONV3,  256, 512, 4, I_C42, -1 },
    { "conv5_2",  L_CONV3,  512, 512, 4, I_C51, -1 },
    { "upv6",     L_DECONV, 512, 256, 3, I_C52, -1 },
    { "conv6_1",  L_CONV3,  512, 256, 3, I_UP6, I_C42 },
    { "conv6_2",  L_CONV3,  256, 256, 3, I_C61, -1 },
    { "upv7",     L_DECONV, 256, 128, 2, I_C62, -1 },
    { "conv7_1",  L_CONV3,  256, 128, 2, I_UP7, I_C32 },
    { "conv7_2",  L_CONV3,  128, 128, 2, I_C71, -1 },
    { "upv8",     L_DECONV, 128,  64, 1, I_C72, -1 },
    { "conv8_1",  L_CONV3,  128,  64, 1, I_UP8, I_C22 },
    { "conv8_2",  L_CONV3,   64,  64, 1, I_C81, -1 },
    { "upv9",     L_DECONV,  64,  32, 0, I_C82, -1 },
    { "conv9_1",  L_CONV3,   64,  32, 0, I_UP9, I_C12 },
    { "conv9_2",  L_CONV3,   32,  32, 0, I_C91, -1 },
    { "conv10_1", L_CONV1,   32,   4, 0, I_C92, -1 },
};
constexpr int kNumLayers = sizeof(kLayers) / sizeof(kLayers[0]);
constexpr int kLevels = 5;       // the frame and the grids of the four 2x2 pools

// An encoder layer behind the skip half of a concat writes channels [cout, 2 cout) of that concat buffer, and the 2x2
// max-pool fused into its tile feeds the next level.
static bool pooled(int l)
{
    for (const LayerSpec& m : kLayers) if (m.skip == l) return true;
    return false;
}

constexpr int kGradBuckets = 4;
// The first layer of each gradient bucket, in backward-completion order; a bucket runs up to the first layer of the one
// before it: upv6..conv10_1, conv5_1..conv5_2, conv2_1..conv4_2, conv1_1..conv1_2.  The last bucket (42 KB) is all that
// is still in flight when backward ends.
constexpr int kBucketFirst[kGradBuckets] = { I_UP6, I_C51, I_C21, I_C11 };
static int bucket_end(int k) { return k == 0 ? kNumLayers : kBucketFirst[k - 1]; }

static_assert(kNumLayers <= kPackMaxEntries, "the packing table (unet_prims.h) holds one entry per layer at most");

// staging [tap][ci][co] -> PyTorch OIHW [co][ci][tap]; one block per (32 co x 32 ci) tile of one layer.  accumulate: add
// the staged gradient to what grads holds (eld_unet_set_accumulate) instead of storing it.  Each element of a layer's
// weight range has one owner thread and no other launch of the step writes that range, so a plain read-modify-write.
__global__ void __launch_bounds__(256)
wgrad_permute_kernel(const float* __restrict__ gtmp, float* __restrict__ grads, const __grid_constant__ PackTable T,
                     int tile_begin, int tile_end, bool accumulate)
{
    // blocks [0, tile_end - tile_begin) move the table tiles [tile_begin, tile_end) (one gradient bucket)
    __shared__ float tile[9][32][33];
    const int gtile = (int)blockIdx.x + tile_begin;
    if (gtile >= tile_end) return;
    int t;
    const PackEntry& e = T.e[find_entry(T, gtile, t)];
    if (e.deconv || !e.perm) return;     // a frozen weight's range of grads is never written
    const int ct = e.cout / 32;
    {
        const int co0 = (t % ct) * 32, ci0 = (t / ct) * 32;
        // 16-byte accesses on both sides (layer offsets are multiples of 4 floats; the staging buffer is 1 KB aligned)
        for (int i = threadIdx.x; i < 9 * 32 * 8; i += 256) {
            const int co4 = i & 7, ci = (i >> 3) & 31, tap = i >> 8;
            const float4 v = __ldg(reinterpret_cast<const float4*>(gtmp + e.src + ((size_t)tap * e.cin + ci0 + ci) * e.cout + co0) + co4);
            float* t4 = &tile[tap][ci][4 * co4];
            t4[0] = v.x; t4[1] = v.y; t4[2] = v.z; t4[3] = v.w;
        }
        __syncthreads();
        if ((reinterpret_cast<uintptr_t>(grads) & 15) == 0) {
            for (int i = threadIdx.x; i < 32 * 72; i += 256) {
                const int co = i / 72, r4 = i - co * 72;           // r = ci*9 + tap, contiguous in OIHW
                float q[4];
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const int r = 4 * r4 + k, ci = r / 9, tap = r - ci * 9;
                    q[k] = tile[tap][ci][co];
                }
                float4* d = reinterpret_cast<float4*>(grads + e.src + ((size_t)(co0 + co) * e.cin + ci0) * 9) + r4;
                if (accumulate) {
                    const float4 p = *d;
                    q[0] += p.x; q[1] += p.y; q[2] += p.z; q[3] += p.w;
                }
                *d = make_float4(q[0], q[1], q[2], q[3]);
            }
        } else {
            for (int i = threadIdx.x; i < 32 * 288; i += 256) {
                const int co = i / 288, r = i - co * 288;
                const int ci = r / 9, tap = r - ci * 9;
                float* d = grads + e.src + ((size_t)(co0 + co) * e.cin + ci0 + ci) * 9 + tap;
                *d = accumulate ? *d + tile[tap][ci][co] : tile[tap][ci][co];
            }
        }
    }
}

}  // namespace eld

using namespace eld;

// Everything a forward leaves for the backward of the same call: activations and concat buffers, pool codes, slope words
// and the packed weights.  layout() places one inside the workspace (the built-in state, eld_unet_forward) or in memory
// the caller owns (eld_unet_forward_state).  The backward writes none of it, so a state stays valid after a backward
// that read it.
struct FwdState {
    __nv_bfloat16* act[kNumLayers] = {};     // the output of each layer that has a buffer of its own
    // slope words (2 bits per element) of the activations whose LeakyReLU' a data gradient applies (training): the dgrad
    // tiles read these instead of the activation itself
    uint32_t* slope[kNumLayers] = {};
    // per level: the concat buffer, and the pooled tensor with its pool codes (1.5 bytes per pooled element, training)
    __nv_bfloat16 *cat[kLevels] = {}, *pool[kLevels] = {}, *code[kLevels] = {};
    __nv_bfloat16* packed = nullptr;
};

struct eld_unet {
    eld_ctx* ctx;
    int n, H, W;
    Layer L[kNumLayers];
    size_t n_params;
    char* ws;
    size_t ws_bytes;
    bool train = false;
    FwdState fs;                 // the built-in forward state, in ws
    // backward scratch (bf16), in ws: the gradient of each layer's output, and per level of the concat buffer (two planar
    // halves, see Runner::conv_dgrad) and of the pooled tensor
    __nv_bfloat16 *dz[kNumLayers] = {}, *dcat[kLevels] = {}, *dp[kLevels] = {};
    float* gtmp = nullptr;
    PackTable table;
    // gradient buckets in backward-completion order (data-parallel overlap, SURVEY 8e): decoder, bottleneck, encoder
    cudaEvent_t bucket_ev[kGradBuckets] = { nullptr, nullptr, nullptr, nullptr };
    int cin0 = 4, cout_last = 4; // channels of the frame in / out: 4 = packed raw, 3 = sRGB (ELD_model.py:377-389)
    int l2_loss = 0;             // 0: nn.L1Loss (the reference default, losses.py:31-32), 1: nn.MSELoss (losses.py:33-34)
    bool accumulate = false;     // eld_unet_train_step adds into grads instead of overwriting it (eld_unet_set_accumulate)
    bool dz1_1_final = false;    // dz1_1 holds the last backward's conv1_1 gradient: set by a backward, cleared by a forward
    // what the backward computes (eld_unet_set_trainable; default: everything).  train_w[l] / train_b[l]: layer l's
    // weight / bias requires grad; wgrad[l]: either does (one launch computes both).  reach[l]: the gradient of layer l's
    // output is needed - l trains, or something upstream of it does (or the frame, when input_grad).  perm_t0 / perm_t1:
    // tile span of the gradient permute per bucket ([kGradBuckets] = the whole table), over the layers that train.
    bool train_w[kNumLayers], train_b[kNumLayers], wgrad[kNumLayers], reach[kNumLayers];
    bool input_grad = true;
    int perm_t0[kGradBuckets + 1], perm_t1[kGradBuckets + 1];
    // optional per-launch profile (CUDA events on the launch stream)
    bool profile = false;
    struct Rec { char name[32]; double flops, bytes; cudaEvent_t e0, e1; };
    std::vector<Rec> recs;
    size_t rec_used = 0;
};

// Places forward state `s` at `base` and, with `scratch`, the backward scratch of `u` (dz, dcat, dp, gtmp) among it in
// the workspace's order; returns the bytes used.  Without `scratch` the state's buffers are packed back to back
// (eld_unet_state_bytes).  train = false: activations and packed weights only.
static size_t layout(eld_unet* u, FwdState* s, char* base, bool train, bool scratch)
{
    size_t off = 0;
    auto take = [&](int lvl, int ch) {       // ch bf16-sized units per pixel of the level's grid
        __nv_bfloat16* p = reinterpret_cast<__nv_bfloat16*>(base + off);
        off += ((size_t)u->n * (u->H >> lvl) * (u->W >> lvl) * ch * 2 + 1023) & ~(size_t)1023;
        return p;
    };
    // activations in state_dict order; a deconv writes into the concat buffer its level's pooled layer placed
    for (int i = 0; i < kNumLayers; ++i) {
        const Layer& l = u->L[i];
        if (l.type == L_CONV1 || l.type == L_DECONV) continue;
        if (!pooled(i)) { s->act[i] = take(l.lvl, l.cout); continue; }
        s->cat[l.lvl] = take(l.lvl, 2 * l.cout);
        s->pool[l.lvl + 1] = take(l.lvl + 1, l.cout);
    }
    if (train && scratch) {       // in the order the backward reaches them
        for (int i = kNumLayers - 1; i >= 0; --i) {
            const Layer& l = u->L[i];
            if (l.type == L_CONV1) continue;
            if (l.type == L_DECONV) { u->dcat[l.lvl] = take(l.lvl, 2 * l.cout); continue; }
            if (pooled(i)) u->dp[l.lvl + 1] = take(l.lvl + 1, l.cout);
            u->dz[i] = take(l.lvl, l.cout);
        }
    }
    if (train) {
        for (int i = 0; i < kNumLayers; ++i)
            if (pooled(i)) s->code[u->L[i].lvl + 1] = take(u->L[i].lvl + 1, u->L[i].cout * 3 / 4);   // 48 B per 32 channels
        // every activation with a buffer of its own, except the head's input: the head applies that LeakyReLU'
        for (int i = 0; i < kNumLayers; ++i) {
            const Layer& l = u->L[i];
            if (l.type == L_CONV3 && !pooled(i) && i != u->L[I_C10].src)
                s->slope[i] = reinterpret_cast<uint32_t*>(take(l.lvl, l.cout / 8));   // cout / 16 words per pixel
        }
    }
    // packed weights
    size_t pk = 0;
    u->L[I_C11].wf_off = pk; pk += 32 * 9 * 32;          // conv1_1: input padded to 32 channels, fprop only
    for (int i = 0; i < kNumLayers; ++i) {
        Layer& l = u->L[i];
        if (i == I_C11 || l.type == L_CONV1) continue;
        const size_t cnt = (size_t)l.cin * l.cout * (l.type == L_CONV3 ? 9 : 4);
        l.wf_off = pk; pk += cnt;
        l.wd_off = pk; pk += cnt;
    }
    s->packed = reinterpret_cast<__nv_bfloat16*>(base + off);
    off += (pk * 2 + 1023) & ~(size_t)1023;
    if (train && scratch) {   // [tap][ci][co] staging of the conv3x3 weight gradients (same offsets as the fp32 parameters)
        u->gtmp = reinterpret_cast<float*>(base + off);
        off += (u->n_params * 4 + 1023) & ~(size_t)1023;
    }
    return off;
}

static void init_layers(eld_unet* u)
{
    size_t off = 0;
    for (int i = 0; i < kNumLayers; ++i) {
        Layer& l = u->L[i];
        static_cast<LayerSpec&>(l) = kLayers[i];
        if (i == 0) l.cin = u->cin0;
        if (i == kNumLayers - 1) l.cout = u->cout_last;
        const size_t ksz = l.type == L_CONV3 ? 9 : (l.type == L_DECONV ? 4 : 1);
        l.w_off = off; off += (size_t)l.cin * l.cout * ksz;
        l.b_off = off; off += l.cout;
        l.wf_off = l.wd_off = 0;
    }
    u->n_params = off;
}

static bool io_ok(int cin, int cout) { return (cin == 3 || cin == 4) && (cout == 3 || cout == 4); }

extern "C" size_t eld_unet_param_count_io(int cin, int cout)
{
    if (!io_ok(cin, cout)) return 0;
    eld_unet tmp{};
    tmp.cin0 = cin; tmp.cout_last = cout;
    init_layers(&tmp);
    return tmp.n_params;
}
extern "C" size_t eld_unet_param_count(void) { return eld_unet_param_count_io(4, 4); }

extern "C" int eld_unet_param_offset_io(const char* name, int is_bias, int cin, int cout, size_t* offset, size_t* count);
extern "C" int eld_unet_param_offset(const char* name, int is_bias, size_t* offset, size_t* count)
{
    return eld_unet_param_offset_io(name, is_bias, 4, 4, offset, count);
}
extern "C" int eld_unet_param_offset_io(const char* name, int is_bias, int cin, int cout, size_t* offset, size_t* count)
{
    ELD_REQUIRE(io_ok(cin, cout), "eld_unet_param_offset: channels in / out must be 3 or 4");
    eld_unet tmp{};
    tmp.cin0 = cin; tmp.cout_last = cout;
    init_layers(&tmp);
    for (int i = 0; i < kNumLayers; ++i) {
        if (strcmp(name, tmp.L[i].name) == 0) {
            const Layer& l = tmp.L[i];
            const size_t ksz = l.type == L_CONV3 ? 9 : (l.type == L_DECONV ? 4 : 1);
            if (offset) *offset = is_bias ? l.b_off : l.w_off;
            if (count) *count = is_bias ? (size_t)l.cout : (size_t)l.cin * l.cout * ksz;
            return ELD_OK;
        }
    }
    set_error("eld_unet_param_offset: unknown layer '%s'", name);
    return ELD_E_ARG;
}

extern "C" size_t eld_unet_workspace_bytes(int n, int h, int w, int train)
{
    eld_unet tmp{};
    tmp.n = n; tmp.H = h; tmp.W = w;
    init_layers(&tmp);
    return layout(&tmp, &tmp.fs, nullptr, train != 0, true) + 1024;
}

extern "C" size_t eld_unet_state_bytes(int n, int h, int w, int cin, int cout)
{
    if (!io_ok(cin, cout) || n <= 0 || h <= 0 || w <= 0) return 0;
    eld_unet tmp{};
    tmp.n = n; tmp.H = h; tmp.W = w; tmp.cin0 = cin; tmp.cout_last = cout;
    init_layers(&tmp);
    return layout(&tmp, &tmp.fs, nullptr, true, false) + 1024;      // + room to align the caller's pointer to 1 KB
}

// The per-launch plan of the backward from the trainable flags (one per parameter tensor, state_dict order), by one
// walk of the forward graph (src / skip) in topological order: a layer's output gradient is needed when the layer
// trains or when the gradient of one of its inputs is.  Runner::backward launches a weight gradient where wgrad[] says
// so and a data gradient towards every input whose producer is reached.
static void derive_needs(eld_unet* u, const uint8_t* flags, bool input_grad)
{
    u->input_grad = input_grad;
    for (int i = 0; i < kNumLayers; ++i) {
        const Layer& l = u->L[i];
        u->train_w[i] = flags[2 * i] != 0;
        u->train_b[i] = flags[2 * i + 1] != 0;
        u->wgrad[i] = u->train_w[i] || u->train_b[i];
        const bool in = l.src < 0 ? input_grad : u->reach[l.src];
        u->reach[i] = u->wgrad[i] || in || (l.skip >= 0 && u->reach[l.skip]);
    }
    // the table holds conv1_2 .. conv9_2 in state_dict order: entry e is layer e + 1
    for (int e = 0; e < u->table.n; ++e) u->table.e[e].perm = u->train_w[e + 1];
    for (int k = 0; k <= kGradBuckets; ++k) {
        const int l0 = k < kGradBuckets ? kBucketFirst[k] : 0, l1 = k < kGradBuckets ? bucket_end(k) : kNumLayers;
        int a = u->table.n, b = 0;
        for (int e = 0; e < u->table.n; ++e)
            if (e + 1 >= l0 && e + 1 < l1 && u->wgrad[e + 1]) { a = a < e ? a : e; b = e + 1; }
        u->perm_t0[k] = a < b ? u->table.tile0[a] : 0;
        u->perm_t1[k] = a < b ? u->table.tile0[b] : 0;
    }
}

extern "C" int eld_unet_create_io(eld_ctx* ctx, int n, int h, int w, int train, void* workspace, size_t bytes,
                                  int cin, int cout, eld_unet** out);
extern "C" int eld_unet_create(eld_ctx* ctx, int n, int h, int w, int train, void* workspace, size_t bytes, eld_unet** out)
{
    return eld_unet_create_io(ctx, n, h, w, train, workspace, bytes, 4, 4, out);
}
extern "C" int eld_unet_create_io(eld_ctx* ctx, int n, int h, int w, int train, void* workspace, size_t bytes,
                                  int cin, int cout, eld_unet** out)
{
    ELD_REQUIRE(ctx && out && workspace, "eld_unet_create: NULL argument");
    ELD_REQUIRE(io_ok(cin, cout), "eld_unet_create: channels in / out must be 3 (sRGB) or 4 (packed raw); got %d -> %d", cin, cout);
    ELD_REQUIRE(n > 0 && h > 0 && w > 0, "eld_unet_create: bad shape");
    ELD_REQUIRE(h % 16 == 0 && w % 16 == 0, "eld_unet_create: H and W must be multiples of 16 (four 2x2 pools, like the reference); got %dx%d", h, w);
    // the head's 32-bit index (launch_head): refused here, before the workspace check, rather than after 23 launches
    ELD_REQUIRE((size_t)n * h * w < kHeadMaxPixels,
                "eld_unet_create: n*H*W = %zu pixels; the head needs fewer than 2^26 (n*H*W*32 < 2^31)", (size_t)n * h * w);
    ELD_CHECK_CUDA(cudaSetDevice(ctx->device));
    ELD_REQUIRE(!train || (h % 128 == 0 && w % 256 == 0),
                "eld_unet_create: TRAINING needs H %% 128 == 0 and W %% 256 == 0 (whole 8x16 / 8x8 gradient tiles at 1/16 scale); got %dx%d", h, w);
    eld_unet* u = new (std::nothrow) eld_unet();
    ELD_REQUIRE(u, "eld_unet_create: out of host memory");
    u->ctx = ctx; u->n = n; u->H = h; u->W = w; u->cin0 = cin; u->cout_last = cout;
    init_layers(u);
    char* base = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(workspace) + 1023) & ~(uintptr_t)1023);
    const size_t need = layout(u, &u->fs, base, train != 0, true) + (base - static_cast<char*>(workspace));
    if (need > bytes) {
        set_error("eld_unet_create: workspace %zu bytes < required %zu", bytes, need);
        delete u;
        return ELD_E_WORKSPACE;
    }
    u->ws = base; u->ws_bytes = bytes; u->train = train != 0;
    int k = 0;
    for (int i = 0; i < kNumLayers; ++i) {
        const Layer& l = u->L[i];
        if (i == I_C11 || l.type == L_CONV1) continue;
        u->table.tile0[k] = k == 0 ? 0 : u->table.tile0[k - 1] + (u->table.e[k - 1].cout / 32) * (u->table.e[k - 1].cin / 32);
        u->table.e[k++] = PackEntry{ l.w_off, l.wf_off, l.wd_off, l.cout, l.cin, l.type == L_DECONV, 1 };
    }
    u->table.tile0[k] = u->table.tile0[k - 1] + (u->table.e[k - 1].cout / 32) * (u->table.e[k - 1].cin / 32);
    u->table.n = k;
    u->table.first_stage = u->n_params;
    u->table.first_dst = u->L[I_C11].w_off;
    u->table.first_wf = u->L[I_C11].wf_off;
    u->table.first_cin = u->cin0;
    {
        uint8_t all[2 * kNumLayers];
        memset(all, 1, sizeof(all));
        derive_needs(u, all, true);
    }
    // conv1_1's operand image: zero once (the packer rewrites all of it every step anyway)
    ELD_CHECK_CUDA(cudaMemset(u->fs.packed + u->L[I_C11].wf_off, 0, 32 * 9 * 32 * sizeof(__nv_bfloat16)));
    // opt in to large dynamic shared memory once (not inside a captured region)
    { int rc = init_gemm_kernels(ctx); if (rc != ELD_OK) { delete u; return rc; } }
    *out = u;
    return ELD_OK;
}

extern "C" void eld_unet_destroy(eld_unet* u)
{
    if (!u) return;
    for (int k = 0; k < kGradBuckets; ++k) if (u->bucket_ev[k]) cudaEventDestroy(u->bucket_ev[k]);
    for (auto& r : u->recs) { cudaEventDestroy(r.e0); cudaEventDestroy(r.e1); }
    delete u;
}

extern "C" int eld_unet_grad_buckets_io(int cin, int cout, size_t* offsets, int max_offsets);
extern "C" int eld_unet_grad_buckets(size_t* offsets, int max_offsets) { return eld_unet_grad_buckets_io(4, 4, offsets, max_offsets); }
extern "C" int eld_unet_grad_buckets_io(int cin, int cout, size_t* offsets, int max_offsets)
{
    ELD_REQUIRE(io_ok(cin, cout), "eld_unet_grad_buckets: channels in / out must be 3 or 4");
    eld_unet tmp{};
    tmp.cin0 = cin; tmp.cout_last = cout;
    init_layers(&tmp);
    if (offsets) {
        ELD_REQUIRE(max_offsets >= 2 * kGradBuckets, "eld_unet_grad_buckets: need room for %d (offset, count) pairs", kGradBuckets);
        for (int k = 0; k < kGradBuckets; ++k) {
            const size_t b = tmp.L[kBucketFirst[k]].w_off;
            const size_t e = bucket_end(k) == kNumLayers ? tmp.n_params : tmp.L[bucket_end(k)].w_off;
            offsets[2 * k] = b; offsets[2 * k + 1] = e - b;
        }
    }
    return kGradBuckets;
}

extern "C" int eld_unet_bucket_events(eld_unet* u, int enable)
{
    ELD_REQUIRE(u, "eld_unet_bucket_events: NULL");
    ELD_CHECK_CUDA(cudaSetDevice(u->ctx->device));
    for (int k = 0; k < kGradBuckets; ++k) {
        if (enable && !u->bucket_ev[k]) ELD_CHECK_CUDA(cudaEventCreateWithFlags(&u->bucket_ev[k], cudaEventDisableTiming));
        if (!enable && u->bucket_ev[k]) { cudaEventDestroy(u->bucket_ev[k]); u->bucket_ev[k] = nullptr; }
    }
    return ELD_OK;
}

extern "C" int eld_unet_wait_bucket(eld_unet* u, int bucket, void* stream)
{
    ELD_REQUIRE(u && bucket >= 0 && bucket < kGradBuckets, "eld_unet_wait_bucket: bad bucket %d", bucket);
    ELD_REQUIRE(u->bucket_ev[bucket], "eld_unet_wait_bucket: call eld_unet_bucket_events(u, 1) before the step");
    ELD_CHECK_CUDA(cudaStreamWaitEvent(static_cast<cudaStream_t>(stream), u->bucket_ev[bucket], 0));
    return ELD_OK;
}

#define TRY(expr) do { int _rc = (expr); if (_rc != ELD_OK) return _rc; } while (0)

namespace {

struct Scope {
    eld_unet* u; cudaStream_t st; eld_unet::Rec* r = nullptr;
    Scope(eld_unet* u_, cudaStream_t st_, const char* layer, const char* what, double flops, double bytes) : u(u_), st(st_)
    {
        if (!u->profile) return;
        if (u->rec_used == u->recs.size()) {
            eld_unet::Rec n{};
            cudaEventCreate(&n.e0); cudaEventCreate(&n.e1);
            u->recs.push_back(n);
        }
        r = &u->recs[u->rec_used++];
        snprintf(r->name, sizeof(r->name), "%s.%s", layer, what);
        r->flops = flops; r->bytes = bytes;
        cudaEventRecord(r->e0, st);
    }
    ~Scope() { if (r) cudaEventRecord(r->e1, st); }
};

struct Runner {
    eld_unet* u;
    const FwdState* s;           // the forward state this call writes (forward) or reads (backward)
    const float* params;
    cudaStream_t st;
    bool accumulate = false;     // the permute adds the conv3x3 weight gradients into grads (an accumulating train step)
    eld_ctx* ctx() const { return u->ctx; }
    const __nv_bfloat16* wf(int i) const { return s->packed + u->L[i].wf_off; }
    const __nv_bfloat16* wd(int i) const { return s->packed + u->L[i].wd_off; }
    const float* bias(int i) const { return params + u->L[i].b_off; }
    // where a weight-gradient launch puts layer li's dW / db: the layer's range of grads when that tensor trains, else the
    // same range of gtmp, which nothing reads.  One launch computes both, so a layer with one frozen tensor still
    // computes it, and the frozen range of grads keeps the zeros of the step's memset.  (A conv3x3's dW is staged in gtmp
    // either way; the permute skips a frozen one.)
    float* dw_to(int li, float* grads) const { return (u->train_w[li] ? grads : u->gtmp) + u->L[li].w_off; }
    float* db_to(int li, float* grads) const { return (u->train_b[li] ? grads : u->gtmp) + u->L[li].b_off; }

    // a tensor as a launch addresses it: base, channel pitch, first channel
    struct View { __nv_bfloat16* p; int pitch, c0; };
    // where layer li writes its output: the concat buffer of its level for a deconv (channels [0, cout)) and for a pooled
    // layer ([cout, 2 cout)), else a buffer of its own
    View out_of(int li) const
    {
        const Layer& l = u->L[li];
        if (l.type == L_DECONV) return { s->cat[l.lvl], 2 * l.cout, 0 };
        if (pooled(li)) return { s->cat[l.lvl], 2 * l.cout, l.cout };
        return { s->act[li], l.cout, 0 };
    }
    // what layer li reads: the whole concat buffer for a concatenating conv, the pooled tensor of a pooled producer, else
    // its producer's output
    View in_of(int li) const
    {
        const Layer& l = u->L[li];
        if (l.skip >= 0) return { s->cat[l.lvl], l.cin, 0 };
        if (pooled(l.src)) return { s->pool[l.lvl], l.cin, 0 };
        return out_of(l.src);
    }

    // a pooled layer's MaxPool2d(2) is fused into the tile's epilogue (pooled tensor has cout channels)
    int conv(int li) const
    {
        const Layer& l = u->L[li];
        const View x = in_of(li), y = out_of(li);
        GemmOp op{};
        op.kind = GEMM_CONV3X3; op.a = x.p; op.a_pitch = x.pitch; op.a_c0 = x.c0; op.cin = l.cin;
        op.n_img = u->n; op.H = u->H >> l.lvl; op.W = u->W >> l.lvl;
        op.b = wf(li); op.cout = l.cout;
        op.act = ACT_LRELU; op.out = y.p; op.out_pitch = y.pitch; op.out_c0 = y.c0; op.bias = bias(li);
        if (pooled(li)) { op.pool_out = s->pool[l.lvl + 1]; op.pool_code = s->code[l.lvl + 1]; }
        op.pool_pitch = l.cout;
        op.slope_out = s->slope[li];
        const double px = (double)u->n * op.H * op.W;
        Scope sc(u, st, l.name, "fprop", 2.0 * px * l.cout * 9 * l.cin, px * 2 * (l.cin + l.cout) + 18.0 * l.cin * l.cout);
        return launch_conv_gemm(ctx(), op, st);
    }
    int deconv(int li) const
    {
        const Layer& l = u->L[li];
        const View x = in_of(li), y = out_of(li);
        GemmOp op{};
        op.kind = GEMM_DECONV; op.a = x.p; op.a_pitch = x.pitch; op.a_c0 = x.c0; op.cin = l.cin;
        op.n_img = u->n; op.H = u->H >> (l.lvl + 1); op.W = u->W >> (l.lvl + 1);
        op.b = wf(li); op.cout = l.cout;
        op.act = ACT_NONE; op.out = y.p; op.out_pitch = y.pitch; op.out_c0 = y.c0; op.bias = bias(li);
        const double px = (double)u->n * op.H * op.W;
        Scope sc(u, st, l.name, "fprop", 2.0 * px * 4 * l.cout * l.cin, px * 2 * (l.cin + 4 * l.cout) + 8.0 * l.cin * l.cout);
        return launch_conv_gemm(ctx(), op, st);
    }
    // data gradient of conv li towards its input, dz [cout] -> [cin]:
    // - a concatenating conv: into the two PLANAR halves of its level's dcat ([up], [skip], pitch cin/2 each) - every
    //   consumer reads exactly one half, and an interleaved buffer made each of them move whole 128-byte lines for 64 useful
    //   bytes (ncu r01: level-1 pool.bwd 570 MB for 300, upv9 dgrad/wgrad 336 MB for 200).  When nothing needs the skip
    //   half (reach[skip]), only the up half's cin/2 columns, read as a row prefix of every block of the same packed operand.
    // - a pooled input: into dp of its level, unmasked (pool_bwd applies the pool code)
    // - else: into the producer's dz, with the LeakyReLU' mask from the producer's slope words
    int conv_dgrad(int li) const
    {
        const Layer& l = u->L[li];
        GemmOp op{};
        int nc = l.cin;
        const bool mask = l.skip < 0 && !pooled(l.src);
        if (l.skip >= 0) {
            op.out = u->dcat[l.lvl]; op.out_pitch = l.cin / 2;
            if (u->reach[l.skip]) {
                op.out2 = skip_half(u->dcat[l.lvl], l.lvl, l.cin / 2); op.out2_pitch = l.cin / 2; op.out_split = l.cin / 2;
            } else {
                nc = l.cin / 2; op.b_block_rows = l.cin <= 256 ? l.cin : 256;
            }
        } else {
            op.out = mask ? u->dz[l.src] : u->dp[l.lvl]; op.out_pitch = l.cin;
        }
        op.kind = GEMM_CONV3X3; op.a = u->dz[li]; op.a_pitch = l.cout; op.a_c0 = 0; op.cin = l.cout;
        op.n_img = u->n; op.H = u->H >> l.lvl; op.W = u->W >> l.lvl;
        op.b = wd(li); op.cout = nc;
        op.act = mask ? ACT_MASK : ACT_NONE; op.out_c0 = 0; op.bias = nullptr;
        op.aux_slope = mask ? s->slope[l.src] : nullptr;
        ELD_REQUIRE(!mask || op.aux_slope, "eld_unet: %s dgrad: no slope words for its LeakyReLU' mask", l.name);
        const double px = (double)u->n * op.H * op.W;
        // the mask is the producer's slope words: two uint32 planes per 32 channels, nc / 4 bytes per pixel
        Scope sc(u, st, l.name, "dgrad", 2.0 * px * l.cout * 9 * nc, px * (2.0 * (nc + l.cout) + (mask ? nc / 4.0 : 0.0)) + 18.0 * nc * l.cout);
        return launch_conv_gemm(ctx(), op, st);
    }
    // data gradient of a deconv: the up half of its level's dcat -> the producer's dz, with its LeakyReLU' mask
    int deconv_dgrad(int li) const
    {
        const Layer& l = u->L[li];
        GemmOp op{};
        op.kind = GEMM_DECONV_DGRAD; op.a = u->dcat[l.lvl]; op.a_pitch = l.cout; op.a_c0 = 0; op.cin = l.cout;
        op.n_img = u->n; op.H = u->H >> (l.lvl + 1); op.W = u->W >> (l.lvl + 1);
        op.b = wd(li); op.cout = l.cin;
        op.act = ACT_MASK; op.out = u->dz[l.src]; op.out_pitch = l.cin; op.out_c0 = 0;
        op.aux_slope = s->slope[l.src];
        ELD_REQUIRE(op.aux_slope, "eld_unet: %s dgrad: no slope words for its LeakyReLU' mask", l.name);
        const double px = (double)u->n * op.H * op.W;
        Scope sc(u, st, l.name, "dgrad", 2.0 * px * 4 * l.cout * l.cin, px * (2.0 * (l.cin + 4 * l.cout) + l.cin / 4.0) + 8.0 * l.cin * l.cout);
        return launch_conv_gemm(ctx(), op, st);
    }
    int conv_wgrad(int li, float* grads) const
    {
        const Layer& l = u->L[li];
        const View x = in_of(li);
        WgradOp op{};
        op.mode = WG_CONV; op.p = x.p; op.p_pitch = x.pitch; op.p_c0 = x.c0; op.p_ch = l.cin;
        op.q = u->dz[li]; op.q_pitch = l.cout; op.q_c0 = 0; op.q_ch = l.cout;
        op.n_img = u->n; op.H = u->H >> l.lvl; op.W = u->W >> l.lvl;
        op.dw = u->gtmp + l.w_off; op.out_tco = 1;
        op.db = db_to(li, grads);                    // bias gradient fused into the same launch
        const double px = (double)u->n * op.H * op.W;
        Scope sc(u, st, l.name, "wgrad", 2.0 * px * l.cout * 9 * l.cin, px * 2 * (l.cin + l.cout) + 36.0 * l.cin * l.cout);
        return launch_wgrad(ctx(), op, st);
    }
    int deconv_wgrad(int li, float* grads) const
    {
        const Layer& l = u->L[li];
        WgradOp op{};
        op.mode = WG_DECONV; op.p = u->dcat[l.lvl]; op.p_pitch = l.cout; op.p_c0 = 0; op.p_ch = l.cout;
        op.q = in_of(li).p; op.q_pitch = l.cin; op.q_c0 = 0; op.q_ch = l.cin;
        op.n_img = u->n; op.H = u->H >> (l.lvl + 1); op.W = u->W >> (l.lvl + 1); op.dw = dw_to(li, grads);
        op.db = db_to(li, grads);                    // bias gradient = column sums of the d(up) boxes, same launch
        const double px = (double)u->n * op.H * op.W;
        Scope sc(u, st, l.name, "wgrad", 2.0 * px * 4 * l.cout * l.cin, px * 2 * (l.cin + 4 * l.cout) + 16.0 * l.cin * l.cout);
        return launch_wgrad(ctx(), op, st);
    }
    // conv1_1's weight gradient: software-im2col tile straight from the fp32 NCHW frame (first_conv.cuh)
    int first_conv_wgrad(const float* x, float* grads) const
    {
        const Layer& l = u->L[I_C11];
        const double px = (double)u->n * u->H * u->W;
        Scope sc(u, st, "conv1_1", "wgrad", 2.0 * px * 32 * 9 * u->cin0, px * (4 * u->cin0 + 64));
        return launch_first_conv_wgrad(ctx(), x, u->cin0, u->dz[I_C11], l.cout, dw_to(I_C11, grads), db_to(I_C11, grads), u->n,
                                       u->H, u->W, st);
    }
    // pooled layer li's pool backward, from the maxima + slope code the forward tile left (the activation is not read
    // again): dp and the PLANAR skip half of the concat gradient -> li's dz
    int pool_bwd(int li) const
    {
        const Layer& l = u->L[li];
        const int lvl = l.lvl + 1, C = l.cout;
        const double pxo = (double)u->n * (u->H >> lvl) * (u->W >> lvl);
        Scope sc(u, st, "pool", "bwd", 0.0, pxo * C * (2 * 9 + 1.5));
        return launch_maxpool_bwd_code(ctx(), s->code[lvl], skip_half(u->dcat[l.lvl], l.lvl, C), C, 0, u->dp[lvl], u->dz[li],
                                       C, u->n, u->H >> lvl, u->W >> lvl, st);
    }
    // second (skip) half of a planar concat gradient: [n][h][w][C] right behind the up half
    __nv_bfloat16* skip_half(__nv_bfloat16* dcat, int lvl, int C) const
    {
        return dcat + (size_t)u->n * (u->H >> lvl) * (u->W >> lvl) * C;
    }
    // the data gradient towards the output of layer li's producer
    int data_grad(int li) const
    {
        const Layer& l = u->L[li];
        if (l.type == L_DECONV) return deconv_dgrad(li);
        TRY(conv_dgrad(li));
        return l.skip < 0 && pooled(l.src) ? pool_bwd(l.src) : ELD_OK;
    }

    // gradients of bucket k are complete in the staging area: move its conv tiles to the PyTorch layout and mark the
    // bucket final (a data-parallel caller all-reduces it on a side stream while the rest of backward runs)
    int finish_bucket(int k, float* g) const
    {
        // Single-GPU steps (no bucket events) move all conv gradients with ONE launch at the end: a permute launch over a
        // few dozen tiles is latency-bound whatever its size, so four of them cost more than one.
        // Data-parallel steps (bucket events on): the bucket's conv gradients move to the PyTorch layout right here, on
        // the compute stream, then an event marks the bucket final.  (Running this permute on the caller's communication
        // stream instead would let it overlap the tiles - any foreign kernel that overlaps the persistent
        // one-CTA-per-SM tiles delays some of their CTAs, and a tile kernel is as slow as its slowest CTA.)
        // Only the span of layers that train is moved, and inside it only the layers whose weight trains (a frozen
        // weight's range of grads keeps the zeros of the memset); a bucket with nothing to move still records its event,
        // so a waiter never sees one from an earlier step.
        const bool per_bucket = u->bucket_ev[0] != nullptr;
        if (!per_bucket && k != kGradBuckets - 1) return ELD_OK;
        const int t0 = u->perm_t0[per_bucket ? k : kGradBuckets];
        const int t1 = u->perm_t1[per_bucket ? k : kGradBuckets];
        if (t1 > t0) {
            Scope sc(u, st, "weights", "gperm", 0.0, 0.0);
            wgrad_permute_kernel<<<t1 - t0, 256, 0, st>>>(u->gtmp, g, u->table, t0, t1, accumulate);
            ELD_CHECK_CUDA(cudaGetLastError());
            count_launch(ctx());
        }
        if (u->bucket_ev[k]) ELD_CHECK_CUDA(cudaEventRecord(u->bucket_ev[k], st));
        return ELD_OK;
    }

    int pack() const
    {
        Scope sc(u, st, "weights", "pack", 0.0, (double)u->n_params * 8);
        return launch_pack(ctx(), params, s->packed, u->table, true, st);
    }

    int forward(const float* x) const
    {
        TRY(pack());
        {
            // conv1_1 (4 -> 32): software-im2col tile straight from the fp32 NCHW frame (first_conv.cuh)
            const double px = (double)u->n * u->H * u->W;
            Scope sc(u, st, "conv1_1", "fprop", 2.0 * px * 32 * 9 * u->cin0, px * (4 * u->cin0 + 64));
            TRY(launch_first_conv(ctx(), x, u->cin0, wf(I_C11), bias(I_C11), s->act[I_C11], u->L[I_C11].cout, u->n, u->H, u->W,
                                  st, s->slope[I_C11]));
        }
        for (int li = I_C11 + 1; li < I_C10; ++li) TRY(u->L[li].type == L_DECONV ? deconv(li) : conv(li));
        return ELD_OK;
    }

    // The layers in reverse state_dict order, each with: its weight gradient if it trains; the finish of the gradient
    // bucket it is the first layer of; the data gradient towards its producer if that one is reached (derive_needs).
    // With every parameter trainable all of them run.
    int backward(const float* x, float* g) const
    {
        int k = 0;                   // the next gradient bucket to finish
        for (int li = I_C10 - 1; li >= I_C11; --li) {
            const Layer& l = u->L[li];
            if (u->wgrad[li])
                TRY(li == I_C11 ? first_conv_wgrad(x, g) : l.type == L_DECONV ? deconv_wgrad(li, g) : conv_wgrad(li, g));
            if (li == kBucketFirst[k]) TRY(finish_bucket(k++, g));
            if (l.src >= 0 && u->reach[l.src]) TRY(data_grad(li));
        }
        return ELD_OK;
    }
};

}  // namespace

// The forward state a call works on: the built-in one (state == NULL), or one laid out in the caller's memory by the
// same layout() (into `tmp`; host-side only)
static const FwdState* state_at(eld_unet* u, void* state, FwdState& tmp)
{
    if (!state) return &u->fs;
    char* base = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(state) + 1023) & ~(uintptr_t)1023);
    layout(u, &tmp, base, true, false);
    return &tmp;
}

extern "C" int eld_unet_forward(eld_unet* u, const float* params, const float* x, float* out, void* stream)
{
    return eld_unet_forward_state(u, nullptr, params, x, out, stream);
}

extern "C" int eld_unet_forward_state(eld_unet* u, void* state, const float* params, const float* x, float* out, void* stream)
{
    ELD_REQUIRE(u && params && x && out, "eld_unet_forward: NULL argument");
    ELD_REQUIRE(!state || u->train, "eld_unet_forward_state: a caller state needs an eld_unet created with train = 1");
    u->dz1_1_final = false;
    ELD_CHECK_CUDA(cudaSetDevice(u->ctx->device));
    FwdState tmp;
    Runner r{ u, state_at(u, state, tmp), params, static_cast<cudaStream_t>(stream) };
    TRY(r.forward(x));
    const double hpx = (double)u->n * u->H * u->W;
    Scope sc(u, r.st, "conv10_1", "fprop", 2.0 * hpx * 128, hpx * (64 + 16));
    return launch_head(u->ctx, r.s->act[I_C92], params + u->L[I_C10].w_off, params + u->L[I_C10].b_off, out, nullptr, nullptr,
                       nullptr, nullptr, nullptr, u->n, (size_t)u->H * u->W, u->cout_last, 0, r.st);
}

extern "C" int eld_unet_train_step(eld_unet* u, const float* params, const float* x, const float* target,
                                   float* out, float* grads, float* loss, void* stream)
{
    ELD_REQUIRE(u && params && x && target && out && grads && loss, "eld_unet_train_step: NULL argument");
    ELD_REQUIRE(u->train, "eld_unet_train_step: the eld_unet was created with train = 0");
    u->dz1_1_final = false;
    ELD_CHECK_CUDA(cudaSetDevice(u->ctx->device));
    Runner r{ u, &u->fs, params, static_cast<cudaStream_t>(stream), u->accumulate };
    if (!u->accumulate) ELD_CHECK_CUDA(cudaMemsetAsync(grads, 0, u->n_params * sizeof(float), r.st));
    ELD_CHECK_CUDA(cudaMemsetAsync(u->gtmp, 0, u->n_params * sizeof(float), r.st));
    ELD_CHECK_CUDA(cudaMemsetAsync(loss, 0, sizeof(float), r.st));
    TRY(r.forward(x));
    {
        // conv10_1 frozen: no dW10 / db10 reduction; nothing below it needed: no dz9_2 (then the step is forward + loss)
        const bool dz = u->reach[I_C92], dw = u->wgrad[I_C10];
        const double hpx = (double)u->n * u->H * u->W;
        Scope sc(u, r.st, "conv10_1", dz || dw ? "fwd+loss+bwd" : "fwd+loss", (dz || dw ? 6.0 : 2.0) * hpx * 128,
                 hpx * (64 + 16 + 16 + (dz ? 64 : 0)));
        TRY(launch_head(u->ctx, u->fs.act[I_C92], params + u->L[I_C10].w_off, params + u->L[I_C10].b_off, out, target,
                        dz ? u->dz[I_C92] : nullptr, dw ? r.dw_to(I_C10, grads) : nullptr,
                        dw ? r.db_to(I_C10, grads) : nullptr, loss, u->n, (size_t)u->H * u->W, u->cout_last, u->l2_loss, r.st));
    }
    TRY(r.backward(x, grads));
    u->dz1_1_final = u->reach[I_C11];
    return ELD_OK;
}

extern "C" int eld_unet_backward(eld_unet* u, const float* params, const float* x, const float* dout, float* grads, void* stream)
{
    return eld_unet_backward_state(u, nullptr, params, x, dout, grads, stream);
}

extern "C" int eld_unet_backward_state(eld_unet* u, void* state, const float* params, const float* x, const float* dout,
                                       float* grads, void* stream)
{
    ELD_REQUIRE(u && params && x && dout && grads, "eld_unet_backward: NULL argument");
    ELD_REQUIRE(u->train, "eld_unet_backward: the eld_unet was created with train = 0");
    ELD_CHECK_CUDA(cudaSetDevice(u->ctx->device));
    FwdState tmp;
    Runner r{ u, state_at(u, state, tmp), params, static_cast<cudaStream_t>(stream) };
    ELD_CHECK_CUDA(cudaMemsetAsync(grads, 0, u->n_params * sizeof(float), r.st));
    ELD_CHECK_CUDA(cudaMemsetAsync(u->gtmp, 0, u->n_params * sizeof(float), r.st));
    if (u->reach[I_C10]) {
        const bool dz = u->reach[I_C92], dw = u->wgrad[I_C10];
        const double hpx = (double)u->n * u->H * u->W;
        Scope sc(u, r.st, "conv10_1", "bwd", 4.0 * hpx * 128, hpx * (64 + 16 + (dz ? 64 : 0)));
        // the head re-forms `out` into scratch (dz1_1 is not written before the very end of backward) and back-propagates dout
        TRY(launch_head(u->ctx, r.s->act[I_C92], params + u->L[I_C10].w_off, params + u->L[I_C10].b_off,
                        reinterpret_cast<float*>(u->dz[I_C11]), dout, dz ? u->dz[I_C92] : nullptr,
                        dw ? r.dw_to(I_C10, grads) : nullptr, dw ? r.db_to(I_C10, grads) : nullptr, nullptr, u->n,
                        (size_t)u->H * u->W, u->cout_last, 2, r.st));
    }
    TRY(r.backward(x, grads));
    u->dz1_1_final = u->reach[I_C11];
    return ELD_OK;
}

extern "C" int eld_unet_set_trainable(eld_unet* u, const uint8_t* flags, int n_flags, int input_grad)
{
    ELD_REQUIRE(u && flags, "eld_unet_set_trainable: NULL argument");
    ELD_REQUIRE(n_flags == 2 * kNumLayers, "eld_unet_set_trainable: %d flags; want %d (weight, bias of every layer in state_dict order)",
                n_flags, 2 * kNumLayers);
    derive_needs(u, flags, input_grad != 0);
    return ELD_OK;
}

extern "C" int eld_unet_input_grad(eld_unet* u, const float* params, float* dx, void* stream)
{
    ELD_REQUIRE(u && params && dx, "eld_unet_input_grad: NULL argument");
    ELD_REQUIRE(u->train, "eld_unet_input_grad: the eld_unet was created with train = 0");
    ELD_REQUIRE(u->dz1_1_final, "eld_unet_input_grad: no eld_unet_backward or eld_unet_train_step since the last forward");
    ELD_CHECK_CUDA(cudaSetDevice(u->ctx->device));
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    const double px = (double)u->n * u->H * u->W;
    Scope sc(u, st, "conv1_1", "dgrad", 2.0 * px * 32 * 9 * u->cin0, px * (64 + 4 * u->cin0));
    return launch_first_conv_dgrad(u->ctx, u->dz[I_C11], params + u->L[I_C11].w_off, u->cin0, dx, u->n, u->H, u->W, st);
}

/* Host-side view of the workspace for tests and debugging: where tensor `name` of the last step lives.  No launch.
   The names come from the layer table: aX_Y / dzX_Y / sign:aX_Y / tie:aX_Y for convX_Y's own output, its gradient and its two planes of slope words;
   catN / dcatN for the concat buffer upvN writes into and its gradient; pN / pcN / ptN / dpN for the pooled tensor at
   level N, its pool codes (maxima and neg words, then the plane of tie words) and its gradient.  Activations belong to the built-in forward state; the gradients are backward scratch. */
extern "C" int eld_unet_buffer(const eld_unet* u, const char* name, void** ptr, int dims[4], int* elem_bytes)
{
    ELD_REQUIRE(u && name && ptr && dims && elem_bytes, "eld_unet_buffer: NULL argument");
    const FwdState& fs = u->fs;
    auto put = [&](const void* p, int n, int h, int w, int units, int eb) {
        *ptr = const_cast<void*>(p); dims[0] = n; dims[1] = h; dims[2] = w; dims[3] = units; *elem_bytes = eb;
        return ELD_OK;
    };
    auto at = [&](const void* p, int lvl, int units, int eb) { return put(p, u->n, u->H >> lvl, u->W >> lvl, units, eb); };
    auto train_only = [&](const void* p, int lvl, int units, int eb) {
        ELD_REQUIRE(u->train, "eld_unet_buffer: '%s' exists only in a training workspace", name);
        return at(p, lvl, units, eb);
    };
    auto pool_ties = [&](const void* code, int lvl, int c) {   // the tie plane behind 32 bytes per (pixel, 32 channels)
        return static_cast<const char*>(code) + (size_t)u->n * (u->H >> lvl) * (u->W >> lvl) * (c / 32) * 32;
    };
    auto is = [name](const char* prefix, const char* id) {     // name == prefix followed by id
        const size_t k = strlen(prefix);
        return strncmp(name, prefix, k) == 0 && strcmp(name + k, id) == 0;
    };
    for (int i = 0; i < kNumLayers; ++i) {
        const Layer& l = u->L[i];
        if (l.type == L_CONV1) continue;
        if (l.type == L_DECONV) {
            if (is("cat", l.name + 3)) return at(fs.cat[l.lvl], l.lvl, 2 * l.cout, 2);
            if (is("dcat", l.name + 3)) return train_only(u->dcat[l.lvl], l.lvl, 2 * l.cout, 2);
            continue;
        }
        if (is("dz", l.name + 4)) return train_only(u->dz[i], l.lvl, l.cout, 2);
        if (pooled(i)) {
            const char pool_lvl[2] = { char('1' + l.lvl), 0 };
            if (is("p", pool_lvl)) return at(fs.pool[l.lvl + 1], l.lvl + 1, l.cout, 2);
            if (is("pc", pool_lvl)) return train_only(fs.code[l.lvl + 1], l.lvl + 1, l.cout, 1);
            if (is("pt", pool_lvl)) return train_only(pool_ties(fs.code[l.lvl + 1], l.lvl + 1, l.cout), l.lvl + 1, l.cout / 2, 1);
            if (is("dp", pool_lvl)) return train_only(u->dp[l.lvl + 1], l.lvl + 1, l.cout, 2);
        } else {
            if (is("a", l.name + 4)) return at(fs.act[i], l.lvl, l.cout, 2);
            if (is("sign:a", l.name + 4) && fs.slope[i]) return at(fs.slope[i], l.lvl, l.cout / 32, 4);
            if (is("tie:a", l.name + 4) && fs.slope[i])
                return at(fs.slope[i] + (size_t)u->n * (u->H >> l.lvl) * (u->W >> l.lvl) * (l.cout / 32), l.lvl, l.cout / 32, 4);
        }
    }
    if (strncmp(name, "sign:", 5) == 0 || strncmp(name, "tie:", 4) == 0) {
        set_error("eld_unet_buffer: no slope words '%s' in this workspace", name);
        return ELD_E_ARG;
    }
    if (strncmp(name, "wf:", 3) == 0 || strncmp(name, "wd:", 3) == 0) {   // packed bf16 operands of one layer
        const bool fprop = name[1] == 'f';
        for (int i = 0; i < kNumLayers; ++i) {
            const Layer& l = u->L[i];
            if (strcmp(name + 3, l.name) != 0 || l.type == L_CONV1 || (i == I_C11 && !fprop)) continue;
            // conv1_1: the [32 co][64 k] K-major image of first_conv.cuh; the others: the operand packed_index describes
            const int count = i == I_C11 ? 32 * 64 : l.cin * l.cout * (l.type == L_CONV3 ? 9 : 4);
            return put(fs.packed + (fprop ? l.wf_off : l.wd_off), 1, 1, 1, count, 2);
        }
        set_error("eld_unet_buffer: no packed operand '%s'", name);
        return ELD_E_ARG;
    }
    if (strcmp(name, "gtmp") == 0) {                 // [tap][ci][co] staging of the conv3x3 weight gradients, parameter offsets
        ELD_REQUIRE(u->train, "eld_unet_buffer: 'gtmp' exists only in a training workspace");
        return put(u->gtmp, 1, 1, 1, (int)u->n_params, 4);
    }
    set_error("eld_unet_buffer: unknown tensor '%s'", name);
    return ELD_E_ARG;
}

extern "C" int eld_adam_step(eld_ctx* ctx, float* params, const float* grads, float* m, float* v, size_t n,
                             float lr, float beta1, float beta2, float eps, float weight_decay, int step,
                             float grad_scale, void* stream)
{
    ELD_REQUIRE(ctx && params && grads && m && v, "eld_adam_step: NULL argument");
    ELD_REQUIRE(step >= 1, "eld_adam_step: step counts from 1");
    ELD_CHECK_CUDA(cudaSetDevice(ctx->device));
    return launch_adam(ctx, params, grads, m, v, n, lr, beta1, beta2, eps, weight_decay, step, grad_scale,
                       static_cast<cudaStream_t>(stream));
}

extern "C" int eld_adam_step_segments(eld_ctx* ctx, float* params, const float* grads, float* m, float* v, const size_t* segs,
                                      const int* steps, int n_segs, float lr, float beta1, float beta2, float eps,
                                      float weight_decay, float grad_scale, void* stream)
{
    ELD_REQUIRE(ctx && params && grads && m && v && (n_segs == 0 || (segs && steps)), "eld_adam_step_segments: NULL argument");
    ELD_CHECK_CUDA(cudaSetDevice(ctx->device));
    AdamHyper hyper[kAdamMaxSegments];                  // every range takes the one set (n_segs > 64 is refused below)
    std::fill(hyper, hyper + kAdamMaxSegments, AdamHyper{ lr, beta1, beta2, eps, weight_decay });
    return launch_adam_segments(ctx, params, grads, m, v, nullptr, segs, steps, hyper, n_segs, grad_scale,
                                static_cast<cudaStream_t>(stream));
}

// a range's hyperparameters as eld_adam_step_ranges(_capturable) accept them (lr only where it is on the host)
static int check_adam_hyper(const char* fn, int s, const float* lr, float beta1, float beta2, float eps, float wd)
{
    ELD_REQUIRE(!lr || (std::isfinite(*lr) && *lr >= 0.f), "%s: range %d: lr %g is not a finite number >= 0", fn, s,
                lr ? (double)*lr : 0.0);
    ELD_REQUIRE(beta1 >= 0.f && beta1 < 1.f && beta2 >= 0.f && beta2 < 1.f, "%s: range %d: betas (%g, %g) outside [0, 1)",
                fn, s, (double)beta1, (double)beta2);
    ELD_REQUIRE(std::isfinite(eps) && eps >= 0.f, "%s: range %d: eps %g is not a finite number >= 0", fn, s, (double)eps);
    ELD_REQUIRE(std::isfinite(wd) && wd >= 0.f, "%s: range %d: weight_decay %g is not a finite number >= 0", fn, s,
                (double)wd);
    return ELD_OK;
}

// a range's ELD_ADAM_* flags: none in the plain records
static unsigned adam_flags(const eld_adam_range&) { return 0; }
static unsigned adam_flags(const eld_adam_range_dev&) { return 0; }
static unsigned adam_flags(const eld_adam_range_ex& r) { return r.flags; }
static unsigned adam_flags(const eld_adam_range_dev_ex& r) { return r.flags; }

// a range's flags as the _ex calls accept them: known bits, and a vmax where AMSGRAD needs one
static int check_adam_flags(const char* fn, int s, unsigned flags, const float* vmax)
{
    ELD_REQUIRE(!(flags & ~(ELD_ADAM_AMSGRAD | ELD_ADAM_MAXIMIZE | ELD_ADAM_DECOUPLED)), "%s: range %d: unknown flags 0x%x",
                fn, s, flags);
    ELD_REQUIRE(vmax || !(flags & ELD_ADAM_AMSGRAD), "%s: range %d: ELD_ADAM_AMSGRAD with a NULL vmax", fn, s);
    return ELD_OK;
}

// eld_adam_step_ranges and its _ex form: every record checked, then one launch_adam_segments
template <class Range>
static int adam_step_ranges(const char* fn, eld_ctx* ctx, float* params, const float* grads, float* m, float* v,
                            float* vmax, const Range* ranges, int n_ranges, float grad_scale, void* stream)
{
    ELD_REQUIRE(ctx && params && grads && m && v && (n_ranges <= 0 || ranges), "%s: NULL argument", fn);
    size_t segs[2 * kAdamMaxSegments];
    int steps[kAdamMaxSegments];
    AdamHyper hyper[kAdamMaxSegments];
    const int k = n_ranges < kAdamMaxSegments ? n_ranges : kAdamMaxSegments;     // more than 64 is refused below
    for (int s = 0; s < k; ++s) {
        const Range& r = ranges[s];
        int rc = check_adam_hyper(fn, s, &r.lr, r.beta1, r.beta2, r.eps, r.weight_decay);
        if (rc == ELD_OK) rc = check_adam_flags(fn, s, adam_flags(r), vmax);
        if (rc != ELD_OK) return rc;
        segs[2 * s] = r.offset; segs[2 * s + 1] = r.count; steps[s] = r.step;
        hyper[s] = AdamHyper{ r.lr, r.beta1, r.beta2, r.eps, r.weight_decay, adam_flags(r) };
    }
    ELD_CHECK_CUDA(cudaSetDevice(ctx->device));
    return launch_adam_segments(ctx, params, grads, m, v, vmax, segs, steps, hyper, n_ranges, grad_scale,
                                static_cast<cudaStream_t>(stream));
}

extern "C" int eld_adam_step_ranges(eld_ctx* ctx, float* params, const float* grads, float* m, float* v,
                                    const eld_adam_range* ranges, int n_ranges, float grad_scale, void* stream)
{
    return adam_step_ranges("eld_adam_step_ranges", ctx, params, grads, m, v, nullptr, ranges, n_ranges, grad_scale,
                            stream);
}

extern "C" int eld_adam_step_ranges_ex(eld_ctx* ctx, float* params, const float* grads, float* m, float* v, float* vmax,
                                       const eld_adam_range_ex* ranges, int n_ranges, float grad_scale, void* stream)
{
    return adam_step_ranges("eld_adam_step_ranges_ex", ctx, params, grads, m, v, vmax, ranges, n_ranges, grad_scale,
                            stream);
}

extern "C" int eld_adam_step_capturable(eld_ctx* ctx, float* params, const float* grads, float* m, float* v, size_t n,
                                        const float* lr, int* step, float beta1, float beta2, float eps, float weight_decay,
                                        float grad_scale, void* stream)
{
    ELD_REQUIRE(ctx && params && grads && m && v && lr && step, "eld_adam_step_capturable: NULL argument");
    ELD_CHECK_CUDA(cudaSetDevice(ctx->device));
    const size_t seg[2] = { 0, n };
    const AdamHyper hyper{ 0.f, beta1, beta2, eps, weight_decay };
    return launch_adam_dev(ctx, params, grads, m, v, nullptr, seg, &step, &lr, &hyper, 1, grad_scale,
                           static_cast<cudaStream_t>(stream));
}

extern "C" int eld_adam_step_segments_capturable(eld_ctx* ctx, float* params, const float* grads, float* m, float* v,
                                                 const size_t* segs, int* const* steps, int n_segs, const float* lr,
                                                 float beta1, float beta2, float eps, float weight_decay, float grad_scale,
                                                 void* stream)
{
    ELD_REQUIRE(ctx && params && grads && m && v && lr && (n_segs == 0 || (segs && steps)),
                "eld_adam_step_segments_capturable: NULL argument");
    ELD_CHECK_CUDA(cudaSetDevice(ctx->device));
    const float* rates[kAdamMaxSegments];               // every range takes the one set (n_segs > 64 is refused below)
    AdamHyper hyper[kAdamMaxSegments];
    std::fill(rates, rates + kAdamMaxSegments, lr);
    std::fill(hyper, hyper + kAdamMaxSegments, AdamHyper{ 0.f, beta1, beta2, eps, weight_decay });
    return launch_adam_dev(ctx, params, grads, m, v, nullptr, segs, steps, rates, hyper, n_segs, grad_scale,
                           static_cast<cudaStream_t>(stream));
}

// eld_adam_step_ranges_capturable and its _ex form: every record checked, then one launch_adam_dev
template <class Range>
static int adam_step_ranges_dev(const char* fn, eld_ctx* ctx, float* params, const float* grads, float* m, float* v,
                                float* vmax, const Range* ranges, int n_ranges, float grad_scale, void* stream)
{
    ELD_REQUIRE(ctx && params && grads && m && v && (n_ranges <= 0 || ranges), "%s: NULL argument", fn);
    size_t segs[2 * kAdamMaxSegments];
    int* steps[kAdamMaxSegments];
    const float* rates[kAdamMaxSegments];
    AdamHyper hyper[kAdamMaxSegments];
    const int k = n_ranges < kAdamMaxSegments ? n_ranges : kAdamMaxSegments;     // more than 64 is refused below
    for (int s = 0; s < k; ++s) {
        const Range& r = ranges[s];
        int rc = check_adam_hyper(fn, s, nullptr, r.beta1, r.beta2, r.eps, r.weight_decay);
        if (rc == ELD_OK) rc = check_adam_flags(fn, s, adam_flags(r), vmax);
        if (rc != ELD_OK) return rc;
        segs[2 * s] = r.offset; segs[2 * s + 1] = r.count; steps[s] = r.step; rates[s] = r.lr;
        hyper[s] = AdamHyper{ 0.f, r.beta1, r.beta2, r.eps, r.weight_decay, adam_flags(r) };
    }
    ELD_CHECK_CUDA(cudaSetDevice(ctx->device));
    return launch_adam_dev(ctx, params, grads, m, v, vmax, segs, steps, rates, hyper, n_ranges, grad_scale,
                           static_cast<cudaStream_t>(stream));
}

extern "C" int eld_adam_step_ranges_capturable(eld_ctx* ctx, float* params, const float* grads, float* m, float* v,
                                               const eld_adam_range_dev* ranges, int n_ranges, float grad_scale,
                                               void* stream)
{
    return adam_step_ranges_dev("eld_adam_step_ranges_capturable", ctx, params, grads, m, v, nullptr, ranges, n_ranges,
                                grad_scale, stream);
}

extern "C" int eld_adam_step_ranges_ex_capturable(eld_ctx* ctx, float* params, const float* grads, float* m, float* v,
                                                  float* vmax, const eld_adam_range_dev_ex* ranges, int n_ranges,
                                                  float grad_scale, void* stream)
{
    return adam_step_ranges_dev("eld_adam_step_ranges_ex_capturable", ctx, params, grads, m, v, vmax, ranges, n_ranges,
                                grad_scale, stream);
}

extern "C" int eld_unet_set_loss(eld_unet* u, int kind)
{
    ELD_REQUIRE(u && (kind == 0 || kind == 1), "eld_unet_set_loss: kind must be 0 (L1) or 1 (MSE)");
    u->l2_loss = kind;
    return ELD_OK;
}

// Gradient accumulation for eld_unet_train_step: with `on`, the step adds its gradients to what grads holds.  The one
// memset of grads is skipped, and the permute adds the staged conv3x3 weight gradients (Runner::finish_bucket, single-GPU
// and per-bucket alike).  Every other writer into grads already adds into it with red.add / atomicAdd:
//   first_conv_kernel<WGRAD>      conv1_1 dW / db      (first_conv.cuh)
//   wgrad_gemm_kernel             deconv dW / db       (wgrad_gemm.cuh)
//   conv3x3_wgrad_thin_kernel     conv3x3 db, fused    (wgrad_thin.cuh; its dW goes to the gtmp staging)
//   head_kernel                   dW10 / db10          (unet_ew.cu)
// A frozen tensor's gradient still goes to gtmp (dw_to / db_to) and the permute skips a frozen conv3x3 weight, so a
// frozen range of grads is never written.  The launches are those of the plain step, in the same order.
// eld_unet_backward / eld_unet_backward_state do not read the flag.
extern "C" int eld_unet_set_accumulate(eld_unet* u, int on)
{
    ELD_REQUIRE(u && u->train, "eld_unet_set_accumulate: needs an eld_unet created with train = 1");
    u->accumulate = on != 0;
    return ELD_OK;
}

extern "C" int eld_clock_probe(eld_ctx* ctx, float* out_mhz_device, void* stream)
{
    ELD_REQUIRE(ctx && out_mhz_device, "eld_clock_probe: NULL argument");
    ELD_CHECK_CUDA(cudaSetDevice(ctx->device));
    return launch_clock_probe(ctx, out_mhz_device, static_cast<cudaStream_t>(stream));
}

extern "C" int eld_unet_profile(eld_unet* u, int enable)
{
    ELD_REQUIRE(u, "eld_unet_profile: NULL");
    u->profile = enable != 0;
    u->rec_used = 0;
    return ELD_OK;
}

/* Synchronises the device; fills up to `max` records of the launches since eld_unet_profile(u, 1). */
extern "C" int eld_unet_profile_read(eld_unet* u, int max, char* names32, float* ms, double* flops, double* bytes, int* count)
{
    ELD_REQUIRE(u && count, "eld_unet_profile_read: NULL");
    ELD_CHECK_CUDA(cudaDeviceSynchronize());
    int n = (int)u->rec_used < max ? (int)u->rec_used : max;
    for (int i = 0; i < n; ++i) {
        float t = 0.f;
        ELD_CHECK_CUDA(cudaEventElapsedTime(&t, u->recs[i].e0, u->recs[i].e1));
        if (names32) memcpy(names32 + 32 * i, u->recs[i].name, 32);
        if (ms) ms[i] = t;
        if (flops) flops[i] = u->recs[i].flops;
        if (bytes) bytes[i] = u->recs[i].bytes;
    }
    *count = n;
    u->rec_used = 0;
    return ELD_OK;
}
