// Network runtime behind include/hv_b200.h: weight ingestion under the reference's state_dict keys, packing into
// kernel layouts, a stack-allocated activation workspace, and the forwards (UNet3DConditionModel, PoseGuider,
// CameraPoseEncoder, AutoencoderKL encode / decode, CLIPVisionModelWithProjection) expressed as sequences of the operators in ops.h.
//
// Activations are channels-last fp16 (N = B*F frames, H, W, C) == a [tokens][C] matrix, so the reference's
// "b c f h w -> (b f) c h w", "(bf) c h w -> (bf) (hw) c" and "(b f) d c -> (b d) f c" rearranges never touch memory:
// spatial tokens are rows, frames of one pixel are rows HW apart.
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <memory>
#include <string>
#include <unordered_map>
#include <tuple>
#include <vector>

#include "../../include/hv_b200.h"
#include "ops.h"

namespace hv {

struct Err {
  int code;
  std::string msg;
};
[[noreturn]] static void fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  throw Err{code, buf};
}
// ck: a CUDA runtime call (copies, memsets, events); ckop: an operator of ops.h
static void ck(cudaError_t e, const char* what) {
  if (e != cudaSuccess) fail(HV_ERR_CUDA, "%s: %s", what, cudaGetErrorString(e));
}
static void ckop(int status, const char* what) {
  if (status != HV_OK) fail(status, "%s: %s", what, last_error());
}
static inline int64_t rup(int64_t a, int64_t b) { return (a + b - 1) / b * b; }

// ------------------------------------------------------------------------------------------ tensors / weights
struct Raw {  // one state_dict entry, fp16 on device
  __half* p = nullptr;
  std::vector<int64_t> shape;
  int64_t numel() const {
    int64_t n = 1;
    for (auto s : shape) n *= s;
    return n;
  }
};

struct Mat {  // packed [rows][cols] fp16
  __half* p = nullptr;
  int64_t rows = 0, cols = 0;
};
struct Norm {
  __half* g = nullptr;
  __half* b = nullptr;
  int C = 0;
  float eps = 1e-5f;
};
struct Lin {
  Mat w;
  __half* bias = nullptr;
  bool geglu = false;  // packed by ff1_geglu: runs with the GEGLU epilogue, w.rows / 2 outputs
  uint8_t* w8 = nullptr;  // FP8 mode: e4m3 copy of w (hv_pack_fp8_rows), one scale per packed row in sw; the linear then runs on e4m3
  float* sw = nullptr;
};
struct Conv3 {       // implicit-GEMM packed 3x3 conv
  Mat w;             // [cout_pad][9 * cin_pad]
  __half* bias = nullptr;  // [cout_pad]
  int cin = 0, cout = 0, cin_pad = 0, cout_pad = 0;
};
struct ConvDirect {  // reference layout (Cout, Cin, 3, 3)
  __half* w = nullptr;
  __half* bias = nullptr;
  int cin = 0, cout = 0;
};

struct Tens {  // channels-last activation
  __half* p = nullptr;
  int NF = 0, H = 0, W = 0, C = 0;
  int64_t rows() const { return static_cast<int64_t>(NF) * H * W; }
  int64_t numel() const { return rows() * C; }
};
struct Q8 {   // e4m3 activation of Tens t's shape (t.p unused): one scale per row (sld == 0) or per (row, 128 columns), s[row * sld + j]
  Tens t;
  uint8_t* q = nullptr;
  float* s = nullptr;
  int sld = 0;
};

struct ResnetW {
  Norm n1, n2;
  Conv3 c1, c2;
  bool has_temb = false;   // UNet resnets add time_emb_proj(silu(emb)) in conv1's epilogue; the VAE's have no time embedding
  Lin temb;
  bool has_sc = false;
  Lin sc;
  int cin = 0, cout = 0;
};
// Self-attention in the layouts of the attention kernels.  dv > d: the spatial kernel, V^T has a ones row per head (h * dv + d, the
// softmax denominator) and zero rows up to dv; dv == d: the single-head d = 512 kernel, no ones row.
struct SelfAttnW {
  Lin qk;                   // [2 * heads * dpad][C] (+ bias): q rows then k rows, each head zero-padded to dpad
  Mat wv;                   // [heads * dv][C]: to_v rows of head h at h * dv, zero rows elsewhere
  __half* vbias = nullptr;  // [heads * dv] row bias of V^T: the ones rows plus to_v's bias at h * dv + j (null when neither exists)
  Lin out;
  int heads = 0, d = 0, dpad = 0, dv = 0;
};
struct SpatialW {
  Norm gn, ln1, ln3;
  Lin proj_in, proj_out;
  SelfAttnW attn1;
  Lin v2, out2;  // cross-attention collapse: to_v (C x xdim), to_out
  Lin ff1, ff2;  // ff1 geglu-packed
  int C = 0;
  int reader_idx = -1;
  // reference bank (B_ref, L, C): `bank` is non-null while a bank is set; its storage (bank_store, bank_cap elements) is kept
  // across hv_clear_ref_banks so that the per-forward clear / set of the Python reader costs no allocation
  __half* bank_store = nullptr;
  int64_t bank_cap = 0;
  __half* bank = nullptr;
  int64_t bank_B = 0, bank_L = 0;
  std::string name;
};
struct TAttnW {
  Norm ln;
  Lin qkv;   // [3C][C], no bias
  Lin out;
  __half* pe = nullptr;  // [max_len][C]
  int max_len = 0;
};
struct TBlockW {   // TemporalTransformerBlock: temporal self-attentions, then LayerNorm -> GEGLU feed-forward + residual
  std::vector<TAttnW> attn;
  Norm ff_norm;
  Lin ff1, ff2;      // ff1 geglu-packed
  int heads = 0, d = 0;
};
struct MotionW {
  Norm gn;
  Lin proj_in, proj_out;
  TBlockW block;
};
struct CamResW {
  Conv3 block1;
  Lin block2;
};
struct ClipLayerW {   // CLIPEncoderLayer: pre-LN self-attention (heads of d = 64, biased q / k / v) and a quick-GELU MLP
  Norm ln1, ln2;
  SelfAttnW attn;
  Lin fc1, fc2;
};

// ------------------------------------------------------------------------------------------ workspace arena
struct Arena {
  uint8_t* base = nullptr;
  size_t cap = 0, off = 0, peak = 0;
  bool dry = false;  // measuring pass: hand out offsets only, launch nothing
  void* alloc(size_t bytes) {
    bytes = (bytes + 1023) & ~size_t(1023);
    if (!dry && off + bytes > cap) fail(HV_ERR_INVALID, "workspace too small: need > %zu bytes, have %zu", off + bytes, cap);
    void* p = base + off;
    off += bytes;
    peak = std::max(peak, off);
    return p;
  }
};
struct Scope {
  Arena& a;
  size_t mark;
  explicit Scope(Arena& ar) : a(ar), mark(ar.off) {}
  ~Scope() { a.off = mark; }
};

}  // namespace hv

using namespace hv;

// ------------------------------------------------------------------------------------------ the model object
struct hv_model {
  hv_config cfg{};
  std::string err;
  std::unordered_map<std::string, Raw> raw;
  std::vector<void*> owned;  // cudaMalloc'ed blocks (weights, banks)
  bool finalized = false;
  cudaStream_t st = nullptr;
  Arena ar;
  void* private_ws = nullptr;
  size_t private_ws_bytes = 0;
  int64_t launches = 0;
  // device-resident timestep (CUDA-graph replay of a denoising loop): t = ts_table[*ts_index] when set
  const long long* ts_table = nullptr;
  const int* ts_index = nullptr;
  // debug taps (per-block parity, error ladder): the activation leaving block `name` of a forward is copied to tap_dst[i] (channels-last
  // fp16, all C channels including any padding), i = the entry of `name` in the plan that the planning pass leaves in tap_list.  A VAE
  // handle plans a decode and then an encode (the decoder's taps, then the encoder's), so a forward finds its entries by name.  With no
  // taps set a forward issues nothing more.
  struct TapInfo { std::string name; int NF, H, W, C; };
  std::vector<TapInfo> tap_list;
  std::vector<void*> tap_dst;
  void tap(const std::string& name, const Tens& t) {
    if (ar.dry) {
      tap_list.push_back({name, t.NF, t.H, t.W, t.C});
      return;
    }
    for (size_t i = 0; i < tap_dst.size() && i < tap_list.size(); ++i) {
      const TapInfo& e = tap_list[i];
      if (e.name != name) continue;
      if (e.NF != t.NF || e.H != t.H || e.W != t.W || e.C != t.C) fail(HV_ERR_STATE, "tap '%s' does not match its plan entry", name.c_str());
      if (tap_dst[i] != nullptr)
        launch(1, {}, [&] { ck(cudaMemcpyAsync(tap_dst[i], t.p, static_cast<size_t>(t.numel()) * 2, cudaMemcpyDeviceToDevice, st), "tap copy"); });
      return;
    }
  }
  // optional per-category device timing (bench.py's roofline): events bracket every categorised operator launch
  enum Cat { CAT_NONE = -1, CAT_GEMM = 0, CAT_CONV = 1, CAT_ATTN = 2, CAT_TATTN = 3, CAT_NORM = 4, CAT_MISC = 5, CAT_N = 6 };
  bool profiling = false;
  struct Rec { int cat; cudaEvent_t a, b; double flops; long long m, n, k; const char* label; };
  std::vector<Rec> recs;
  std::vector<cudaEvent_t> ev_pool;
  size_t ev_used = 0;
  cudaEvent_t ev() {
    if (ev_used == ev_pool.size()) {
      cudaEvent_t e;
      ck(cudaEventCreate(&e), "cudaEventCreate");
      ev_pool.push_back(e);
    }
    return ev_pool[ev_used++];
  }
  // the profile row of one operator; CAT_NONE: counted, not timed
  struct Op { int cat = CAT_NONE; const char* label = ""; double flops = 0; long long M = 0, N = 0, K = 0; };
  // The one path of device work in a forward: fn issues `n` launches (kernels, memsets, copies).  The planning pass only sizes the
  // workspace (ar.base is null), so nothing is issued in it.
  template <class Fn> void launch(int n, const Op& op, Fn&& fn) {
    if (ar.dry) return;
    launches += n;
    if (!profiling || op.cat == CAT_NONE) {
      fn();
      return;
    }
    cudaEvent_t a = ev();
    cudaEventRecord(a, st);
    fn();
    cudaEvent_t b = ev();
    cudaEventRecord(b, st);
    recs.push_back({op.cat, a, b, op.flops, op.M, op.N, op.K, op.label});
  }

  // ---- UNet
  Conv3 conv_in;  // 4 input channels zero-padded to 64: runs on the implicit-GEMM kernel
  Lin te1, te2;
  // down_blocks.i / mid_block / up_blocks.i: layer j is res[j], then attn[j] and mm[j] where present, and the stage ends in an
  // optional down- or up-sampler conv
  struct Stage {
    std::string name;
    std::vector<ResnetW> res;
    std::vector<SpatialW> attn;
    std::vector<MotionW> mm;
    bool has_sampler = false;
    Conv3 sampler;
  };
  std::vector<Stage> down, up;
  Stage mid;
  Norm norm_out;
  Conv3 conv_out;
  std::vector<SpatialW*> readers;  // reference-bank order
  __half* const* bank_out = nullptr;  // writer forward: reader-order destinations of every block's LayerNorm-1 output (the "bank")
  // ---- PoseGuider
  ConvDirect pg_in;
  std::vector<Conv3> pg_convs;  // blocks.0..5, conv_out
  std::vector<int> pg_strides;
  std::vector<bool> pg_small;   // layer runs on the small-channel mma.sync kernel at its true channel counts (smallconv.cu)
  bool pg_fast_in = false;      // conv_in reads the (B,3,F,H,W) image directly and writes 16 channels (no layout pass, no padding)
  // ---- CameraPoseEncoder
  Conv3 cam_in;
  std::vector<CamResW> cam_res;
  std::vector<TBlockW> cam_att;
  Lin cam_zero;
  // ---- AutoencoderKL: encoder.* / decoder.* (the down / up blocks and the mid block's two resnets are Stages without attention)
  struct VaeHalf {
    Conv3 conv_in;
    std::vector<Stage> blocks;
    Stage mid;
    Norm attn_gn;    // the mid-block attention: GroupNorm, then one head of C = 512 channels with biased q / k / v
    SelfAttnW attn;
    Norm norm_out;
    Conv3 conv_out;
  };
  VaeHalf enc, dec;
  Lin quant, post_quant;   // post_quant_conv zero-padded to [64][64]: its output is conv_in's 64-channel padded input
  // ---- CLIPVisionModelWithProjection
  static constexpr int kClipHeadDim = 64;
  Lin clip_patch;          // patch_embedding flattened to [hidden][3 p^2] and zero-padded to [hidden][Kpad] (no bias)
  __half* clip_cls = nullptr;   // class_embedding [hidden]
  __half* clip_pos = nullptr;   // position_embedding [1 + (S/p)^2][hidden]
  Norm clip_pre, clip_post;
  std::vector<ClipLayerW> clip_layers;
  Mat clip_proj;           // visual_projection [projection_dim][hidden]

  ~hv_model() {
    for (void* p : owned) cudaFree(p);
    if (private_ws) cudaFree(private_ws);
    for (auto e : ev_pool) cudaEventDestroy(e);
  }

  // ================================================================== weight helpers
  __half* dmalloc(int64_t halves) {
    void* p = nullptr;
    ck(cudaMalloc(&p, static_cast<size_t>(halves) * 2), "cudaMalloc(weights)");
    owned.push_back(p);
    return static_cast<__half*>(p);
  }
  const Raw& get(const std::string& key) {
    auto it = raw.find(key);
    if (it == raw.end()) fail(HV_ERR_MISSING, "missing weight '%s'", key.c_str());
    return it->second;
  }
  bool has(const std::string& key) const { return raw.count(key) != 0; }

  __half* vec(const std::string& key, int64_t n, int64_t pad_to = 0) {
    const Raw& r = get(key);
    if (r.numel() != n) fail(HV_ERR_INVALID, "weight '%s' has %lld elements, expected %lld", key.c_str(), (long long)r.numel(), (long long)n);
    if (pad_to <= n) return r.p;
    __half* p = dmalloc(pad_to);
    ck(cudaMemsetAsync(p, 0, pad_to * 2, st), "memset");
    ck(cudaMemcpyAsync(p, r.p, n * 2, cudaMemcpyDeviceToDevice, st), "memcpy");
    return p;
  }
  Norm norm(const std::string& pfx, int C, float eps) {
    Norm n;
    n.g = vec(pfx + ".weight", C);
    n.b = vec(pfx + ".bias", C);
    n.C = C;
    n.eps = eps;
    return n;
  }
  Mat mat(const std::string& key, int64_t rows, int64_t cols) {  // 2-D (or 4-D 1x1 conv) weight used as is
    const Raw& r = get(key);
    if (r.numel() != rows * cols) fail(HV_ERR_INVALID, "weight '%s': %lld elements, expected %lld x %lld", key.c_str(), (long long)r.numel(), (long long)rows, (long long)cols);
    return Mat{r.p, rows, cols};
  }
  Lin lin(const std::string& pfx, int64_t out, int64_t in, bool bias = true) {
    Lin l;
    l.w = mat(pfx + ".weight", out, in);
    if (bias) l.bias = vec(pfx + ".bias", out);
    return l;
  }
  const Raw& conv3_weight(const std::string& pfx, int cout, int cin) {
    const Raw& r = get(pfx + ".weight");
    if (r.shape.size() != 4 || r.shape[0] != cout || r.shape[1] != cin || r.shape[2] != 3 || r.shape[3] != 3)
      fail(HV_ERR_INVALID, "weight '%s.weight' is not (%d,%d,3,3)", pfx.c_str(), cout, cin);
    return r;
  }
  // Channel padding of a packed [cout_pad][9 * cin_pad] 3x3 conv.  The implicit-GEMM kernel reads 64-channel k-blocks and writes
  // cout rounded up to 8 (PAD_OUT_64: to 64, the output feeds another implicit-GEMM conv); the small-channel kernel (smallconv.cu)
  // takes the true channel counts (PAD_NONE).
  enum ConvPad { PAD_GEMM, PAD_OUT_64, PAD_NONE };
  Conv3 conv3(const std::string& pfx, int cout, int cin, ConvPad pad = PAD_GEMM) {
    const Raw& r = conv3_weight(pfx, cout, cin);
    Conv3 c;
    c.cin = cin;
    c.cout = cout;
    c.cin_pad = pad == PAD_NONE ? cin : static_cast<int>(rup(cin, 64));
    c.cout_pad = pad == PAD_NONE ? cout : static_cast<int>(rup(cout, pad == PAD_OUT_64 ? 64 : 8));
    c.w.rows = c.cout_pad;
    c.w.cols = 9LL * c.cin_pad;
    c.w.p = dmalloc(c.w.rows * c.w.cols);
    ckop(op_pack_conv3x3(r.p, c.w.p, cout, cin, c.cout_pad, c.cin_pad, st), "pack conv3x3");
    c.bias = vec(pfx + ".bias", cout, c.cout_pad);
    return c;
  }
  // Upsample3D's conv packed for op_upconv2x2: [4 parities][cout][4 * cin]
  Conv3 upconv(const std::string& pfx, int cout, int cin) {
    const Raw& r = conv3_weight(pfx, cout, cin);
    if ((cin % 64) || (cout % 8)) fail(HV_ERR_INVALID, "upsampler conv '%s': %d -> %d channels must be multiples of 64 / 8", pfx.c_str(), cin, cout);
    Conv3 c;
    c.cin = c.cin_pad = cin;
    c.cout = c.cout_pad = cout;
    c.w.rows = 4LL * cout;
    c.w.cols = 4LL * cin;
    c.w.p = dmalloc(c.w.rows * c.w.cols);
    ckop(op_pack_upconv2x2(r.p, c.w.p, cout, cin, st), "pack upconv2x2");
    c.bias = vec(pfx + ".bias", cout);
    return c;
  }
  ConvDirect conv_direct(const std::string& pfx, int cout, int cin) {
    ConvDirect c;
    c.w = get(pfx + ".weight").p;
    c.bias = vec(pfx + ".bias", cout);
    c.cin = cin;
    c.cout = cout;
    return c;
  }
  Lin ff1_geglu(const std::string& pfx, int C) {  // net.0.proj: [8C][C] + bias -> 128-row hidden/gate interleave
    const Raw& w = get(pfx + ".weight");
    const Raw& b = get(pfx + ".bias");
    if (w.numel() != 8LL * C * C || b.numel() != 8LL * C) fail(HV_ERR_INVALID, "'%s' is not a GEGLU proj of dim %d", pfx.c_str(), C);
    if ((4 * C) % 128) fail(HV_ERR_INVALID, "GEGLU inner dim %d must be a multiple of 128", 4 * C);
    Lin l;
    l.w = Mat{dmalloc(8LL * C * C), 8LL * C, C};
    ckop(op_pack_geglu(w.p, l.w.p, 8 * C, C, st), "pack geglu");
    l.bias = dmalloc(8LL * C);
    ckop(op_pack_geglu(b.p, l.bias, 8 * C, 1, st), "pack geglu bias");
    l.geglu = true;
    return l;
  }
  // FP8 mode (hv_config.fp8_linears): the transformer feed-forwards LN -> FF1 -> FF2 of width C >= 1280 run on e4m3.  They are the only
  // covered shapes measured faster than fp16 (DESIGN.md §9); every other linear stays fp16.  The camera encoder and the other networks
  // have no FP8 mode.
  bool fp8_ff(int C) const { return cfg.kind == HV_KIND_UNET3D && cfg.fp8_linears && C >= 1280; }
  void add_fp8(Lin& l) {
    l.w8 = reinterpret_cast<uint8_t*>(dmalloc((l.w.rows * l.w.cols + 1) / 2));
    l.sw = reinterpret_cast<float*>(dmalloc(2 * l.w.rows));
    ckop(op_pack_fp8_rows(l.w.p, l.w8, l.sw, l.w.rows, l.w.cols, st), "pack fp8 rows");
  }

  // temb == 0: a resnet without time embedding (no time_emb_proj)
  ResnetW resnet(const std::string& pfx, int cin, int cout, int temb, float eps = 1e-5f) {
    ResnetW r;
    r.cin = cin;
    r.cout = cout;
    r.n1 = norm(pfx + ".norm1", cin, eps);
    r.c1 = conv3(pfx + ".conv1", cout, cin);
    r.has_temb = temb > 0;
    if (r.has_temb) r.temb = lin(pfx + ".time_emb_proj", cout, temb);
    r.n2 = norm(pfx + ".norm2", cout, eps);
    r.c2 = conv3(pfx + ".conv2", cout, cout);
    r.has_sc = cin != cout;
    if (r.has_sc) r.sc = lin(pfx + ".conv_shortcut", cout, cin);
    return r;
  }
  // [heads * dv]: 1 at row h * dv + d (the softmax-denominator row of every head of V^T), else 0
  __half* vones(int heads, int dv, int d) {
    std::vector<__half> ones(static_cast<size_t>(heads) * dv, __float2half(0.f));
    for (int hh = 0; hh < heads; ++hh) ones[static_cast<size_t>(hh) * dv + d] = __float2half(1.f);
    __half* p = dmalloc(static_cast<int64_t>(ones.size()));
    ck(cudaMemcpyAsync(p, ones.data(), ones.size() * 2, cudaMemcpyHostToDevice, st), "vones upload");
    ck(cudaStreamSynchronize(st), "vones sync");  // `ones` is a host temporary
    return p;
  }
  // The projections `keys` ([heads * d][cols] each; cols = 1 for biases) stacked into one matrix: head h of keys[i] at rows
  // (i * heads + h) * dpad .., zero rows from d to dpad
  __half* stack_heads(const std::vector<std::string>& keys, int heads, int d, int dpad, int cols) {
    const int64_t rows = static_cast<int64_t>(heads) * dpad;
    __half* p = dmalloc(static_cast<int64_t>(keys.size()) * rows * cols);
    for (size_t i = 0; i < keys.size(); ++i)
      ckop(op_pack_heads(mat(keys[i], static_cast<int64_t>(heads) * d, cols).p, p + i * rows * cols, heads, d, dpad, cols, st), "pack heads");
    return p;
  }
  // q / k / v / out: key prefixes of the projections; bias: q, k and v have biases (out always has one)
  SelfAttnW self_attn(const std::string& q, const std::string& k, const std::string& v, const std::string& out, int C, int heads, bool bias) {
    SelfAttnW a;
    a.heads = heads;
    a.d = C / heads;
    a.dpad = static_cast<int>(rup(a.d, 16));
    a.dv = (a.d == 512 && heads == 1) ? a.d : static_cast<int>(rup(a.d + 1, 16));
    a.qk.w = Mat{stack_heads({q + ".weight", k + ".weight"}, heads, a.d, a.dpad, C), 2LL * heads * a.dpad, C};
    if (bias) a.qk.bias = stack_heads({q + ".bias", k + ".bias"}, heads, a.d, a.dpad, 1);
    a.wv = Mat{stack_heads({v + ".weight"}, heads, a.d, a.dv, C), static_cast<int64_t>(heads) * a.dv, C};
    if (a.dv > a.d) a.vbias = vones(heads, a.dv, a.d);
    else if (bias) a.vbias = dmalloc(static_cast<int64_t>(heads) * a.dv);
    if (bias)
      ck(cudaMemcpy2DAsync(a.vbias, static_cast<size_t>(a.dv) * 2, vec(v + ".bias", C), static_cast<size_t>(a.d) * 2, static_cast<size_t>(a.d) * 2, heads,
                           cudaMemcpyDeviceToDevice, st), "v bias pack");
    a.out = lin(out, C, C);
    return a;
  }
  SpatialW spatial(const std::string& pfx, int C) {
    SpatialW s;
    s.name = pfx;
    s.C = C;
    const int d = C / cfg.heads;
    if (d % 8) fail(HV_ERR_INVALID, "head dim %d (C=%d / %d heads) must be a multiple of 8", d, C, cfg.heads);
    s.gn = norm(pfx + ".norm", C, 1e-6f);
    s.proj_in = lin(pfx + ".proj_in", C, C);
    s.proj_out = lin(pfx + ".proj_out", C, C);
    const std::string b = pfx + ".transformer_blocks.0";
    s.ln1 = norm(b + ".norm1", C, 1e-5f);
    s.ln3 = norm(b + ".norm3", C, 1e-5f);
    const std::string a = b + ".attn1";
    s.attn1 = self_attn(a + ".to_q", a + ".to_k", a + ".to_v", a + ".to_out.0", C, cfg.heads, false);
    s.v2 = lin(b + ".attn2.to_v", C, cfg.cross_attention_dim, false);
    s.out2 = lin(b + ".attn2.to_out.0", C, C);
    s.ff1 = ff1_geglu(b + ".ff.net.0.proj", C);
    s.ff2 = lin(b + ".ff.net.2", C, 4 * C);
    if (fp8_ff(C)) { add_fp8(s.ff1); add_fp8(s.ff2); }
    return s;
  }
  TAttnW tattn(const std::string& attn_pfx, const std::string& norm_pfx, int C) {
    TAttnW t;
    t.ln = norm(norm_pfx, C, 1e-5f);
    t.qkv.w = Mat{stack_heads({attn_pfx + ".to_q.weight", attn_pfx + ".to_k.weight", attn_pfx + ".to_v.weight"}, 1, C, C, C), 3LL * C, C};
    t.out = lin(attn_pfx + ".to_out.0", C, C);
    const Raw& pe = get(attn_pfx + ".pos_encoder.pe");
    if (pe.numel() % C) fail(HV_ERR_INVALID, "'%s.pos_encoder.pe' width != %d", attn_pfx.c_str(), C);
    t.pe = pe.p;
    t.max_len = static_cast<int>(pe.numel() / C);
    return t;
  }
  // TemporalTransformerBlock `pfx` with n_attn temporal self-attentions
  TBlockW tblock(const std::string& pfx, int C, int heads, int n_attn) {
    TBlockW b;
    b.heads = heads;
    b.d = C / heads;
    for (int i = 0; i < n_attn; ++i)
      b.attn.push_back(tattn(pfx + ".attention_blocks." + std::to_string(i), pfx + ".norms." + std::to_string(i), C));
    b.ff_norm = norm(pfx + ".ff_norm", C, 1e-5f);
    b.ff1 = ff1_geglu(pfx + ".ff.net.0.proj", C);
    b.ff2 = lin(pfx + ".ff.net.2", C, 4 * C);
    if (fp8_ff(C)) { add_fp8(b.ff1); add_fp8(b.ff2); }
    return b;
  }
  MotionW motion(const std::string& pfx, int C) {
    MotionW m;
    const std::string t = pfx + ".temporal_transformer";
    m.gn = norm(t + ".norm", C, 1e-6f);
    m.proj_in = lin(t + ".proj_in", C, C);
    m.proj_out = lin(t + ".proj_out", C, C);
    m.block = tblock(t + ".transformer_blocks.0", C, cfg.heads, 2);
    return m;
  }

  // layer j: a resnet ins[j] -> C channels (GroupNorm eps), then a transformer if j < n_attn and a motion module if j < n_mm
  Stage stage(const std::string& name, const std::vector<int>& ins, int C, int temb, size_t n_attn, size_t n_mm, float eps = 1e-5f) {
    Stage s;
    s.name = name;
    for (size_t j = 0; j < ins.size(); ++j) {
      const std::string sj = "." + std::to_string(j);
      s.res.push_back(resnet(name + ".resnets" + sj, ins[j], C, temb, eps));
      if (j < n_attn) s.attn.push_back(spatial(name + ".attentions" + sj, C));
      if (j < n_mm) s.mm.push_back(motion(name + ".motion_modules" + sj, C));
    }
    return s;
  }

  void build_unet() {
    const int* ch = cfg.block_out_channels;
    const int temb = ch[0] * 4;
    const bool mm = cfg.use_motion_module != 0;
    conv_in = conv3("conv_in", ch[0], cfg.in_channels);
    te1 = lin("time_embedding.linear_1", temb, ch[0]);
    te2 = lin("time_embedding.linear_2", temb, temb);
    down.clear();
    up.clear();
    int prev = ch[0];
    for (int i = 0; i < 4; ++i) {
      Stage s = stage("down_blocks." + std::to_string(i), {prev, ch[i]}, ch[i], temb, i < 3 ? 2 : 0, mm ? 2 : 0);
      s.has_sampler = i < 3;
      if (s.has_sampler) s.sampler = conv3(s.name + ".downsamplers.0.conv", ch[i], ch[i]);
      down.push_back(std::move(s));
      prev = ch[i];
    }
    mid = stage("mid_block", {ch[3], ch[3]}, ch[3], temb, 1, (mm && !cfg.no_mid_motion_module) ? 1 : 0);
    const int rev[4] = {ch[3], ch[2], ch[1], ch[0]};
    prev = rev[0];
    for (int i = 0; i < 4; ++i) {
      const int c = rev[i], skip = rev[std::min(i + 1, 3)];   // resnet j reads h ++ the j-th skip from the end
      Stage s = stage("up_blocks." + std::to_string(i), {prev + c, c + c, c + skip}, c, temb, i > 0 ? 3 : 0, mm ? 3 : 0);
      s.has_sampler = i < 3;
      if (s.has_sampler) s.sampler = upconv(s.name + ".upsamplers.0.conv", c, c);
      up.push_back(std::move(s));
      prev = c;
    }
    if (cfg.kind == HV_KIND_UNET3D) {   // the reference ("writer") 2-D UNet has its post-process removed (unet_2d_condition.py:1295-1299)
      norm_out = norm("conv_norm_out", ch[0], 1e-5f);
      conv_out = conv3("conv_out", cfg.out_channels, ch[0]);
    }
    // reader order: DFS(down_blocks, up_blocks, mid_block), stable sort by descending width
    readers.clear();
    for (auto& d : down) for (auto& a : d.attn) readers.push_back(&a);
    for (auto& u : up) for (auto& a : u.attn) readers.push_back(&a);
    for (auto& a : mid.attn) readers.push_back(&a);
    std::stable_sort(readers.begin(), readers.end(), [](const SpatialW* x, const SpatialW* y) { return x->C > y->C; });
    for (size_t i = 0; i < readers.size(); ++i) readers[i]->reader_idx = static_cast<int>(i);
  }

  void build_pose_guider() {
    const int* bc = cfg.pg_block_channels;
    pg_in = conv_direct("conv_in", bc[0], cfg.pg_cond_channels);
    pg_convs.clear();
    pg_strides.clear();
    pg_small.clear();
    // the 16 / 32-channel layers at (up to) full image resolution are HBM-bound: they run at their true channel counts on the small-channel
    // kernel as long as the chain from conv_in is unbroken; from the first layer it does not cover, the wgmma implicit GEMM takes over
    pg_fast_in = cfg.pg_cond_channels == 3 && bc[0] == 16 && smallconv_supported(bc[0], bc[0], 1);
    bool chain = pg_fast_in;
    for (int i = 0; i < 3; ++i) {
      for (int k = 0; k < 2; ++k) {
        const int cin = bc[i], cout = k == 0 ? bc[i] : bc[i + 1], stride = k == 0 ? 1 : 2;
        const std::string name = "blocks." + std::to_string(2 * i + k);
        chain = chain && smallconv_supported(cin, cout, stride);
        pg_small.push_back(chain);
        pg_convs.push_back(conv3(name, cout, cin, chain ? PAD_NONE : PAD_OUT_64));
        pg_strides.push_back(stride);
      }
    }
    pg_convs.push_back(conv3("conv_out", cfg.pg_out_channels, bc[3]));
    pg_strides.push_back(1);
    pg_small.push_back(false);
  }

  void build_camera() {
    const int C = cfg.cam_channels;
    cam_in = conv3("encoder_conv_in", C, cfg.cam_cin);
    for (int j = 0; j < cfg.cam_nums_rb; ++j) {
      const std::string p = "encoder_down_conv_blocks.0." + std::to_string(j);
      CamResW r;
      r.block1 = conv3(p + ".block1", C, C);
      r.block2 = lin(p + ".block2", C, C);
      cam_res.push_back(r);
      cam_att.push_back(tblock("encoder_down_attention_blocks.0." + std::to_string(j), C, cfg.cam_heads, 1));
    }
    cam_zero = lin("zero_conv_layers.0", C, C, false);
  }

  // ---- AutoencoderKL (diffusers 0.24 key names; SD layout: 4 levels, 2 resnets per encoder level, 3 per decoder level)
  // [n_pad][k_pad] zero-padded copy of an [n][k] linear / 1x1 conv weight, bias (if any) zero-padded to n_pad
  Lin padded_linear(const std::string& pfx, int n, int k, int n_pad, int k_pad, bool bias = true) {
    const Raw& w = get(pfx + ".weight");
    if (w.numel() != static_cast<int64_t>(n) * k) fail(HV_ERR_INVALID, "weight '%s.weight' has %lld elements, expected %d x %d", pfx.c_str(), (long long)w.numel(), n, k);
    Lin l;
    l.w = Mat{dmalloc(static_cast<int64_t>(n_pad) * k_pad), n_pad, k_pad};
    ck(cudaMemsetAsync(l.w.p, 0, static_cast<size_t>(n_pad) * k_pad * 2, st), "memset");
    ck(cudaMemcpy2DAsync(l.w.p, static_cast<size_t>(k_pad) * 2, w.p, static_cast<size_t>(k) * 2, static_cast<size_t>(k) * 2, n, cudaMemcpyDeviceToDevice, st),
       "padded weight copy");
    if (bias) l.bias = vec(pfx + ".bias", n, n_pad);
    return l;
  }
  // the mid block's attention (and its GroupNorm) of half `pfx`
  void vae_attn(VaeHalf& v, const std::string& pfx, int C) {
    if (C != 512) fail(HV_ERR_INVALID, "'%s': the mid-block attention is implemented for 512 channels (one head of d = 512), got %d", pfx.c_str(), C);
    v.attn_gn = norm(pfx + ".group_norm", C, 1e-6f);
    v.attn = self_attn(pfx + ".to_q", pfx + ".to_k", pfx + ".to_v", pfx + ".to_out.0", C, 1, true);
  }
  void build_vae() {
    const int* ch = cfg.block_out_channels;
    const int zc = cfg.vae_latent_channels;
    if (zc <= 0 || zc > 64 || (2 * zc) % 8) fail(HV_ERR_INVALID, "vae_latent_channels = %d: 2 * latent channels must be a multiple of 8 and <= 128", zc);
    if (cfg.in_channels <= 0 || cfg.in_channels > 64 || cfg.out_channels <= 0 || cfg.out_channels > 64)
      fail(HV_ERR_INVALID, "AutoencoderKL image channels (%d in, %d out) must be 1..64", cfg.in_channels, cfg.out_channels);
    // encoder: conv_in, 4 x DownEncoderBlock2D (the first three end in Downsample2D: pad (0, 1, 0, 1) + stride-2 conv), mid block,
    // conv_norm_out + SiLU, conv_out -> 2 * latent channels (mean | logvar)
    enc.conv_in = conv3("encoder.conv_in", ch[0], cfg.in_channels);
    enc.blocks.clear();
    int prev = ch[0];
    for (int i = 0; i < 4; ++i) {
      Stage s = stage("encoder.down_blocks." + std::to_string(i), {prev, ch[i]}, ch[i], 0, 0, 0, 1e-6f);
      s.has_sampler = i < 3;
      if (s.has_sampler) s.sampler = conv3(s.name + ".downsamplers.0.conv", ch[i], ch[i]);
      enc.blocks.push_back(std::move(s));
      prev = ch[i];
    }
    enc.mid = stage("encoder.mid_block", {ch[3], ch[3]}, ch[3], 0, 0, 0, 1e-6f);
    vae_attn(enc, "encoder.mid_block.attentions.0", ch[3]);
    enc.norm_out = norm("encoder.conv_norm_out", ch[3], 1e-6f);
    enc.conv_out = conv3("encoder.conv_out", 2 * zc, ch[3]);
    quant = lin("quant_conv", 2 * zc, 2 * zc);
    // decoder: post_quant_conv, conv_in, mid block, 4 x UpDecoderBlock2D over (ch3, ch2, ch1, ch0) (the first three end in nearest 2x +
    // 3x3 conv), conv_norm_out + SiLU, conv_out
    post_quant = padded_linear("post_quant_conv", zc, zc, 64, 64);
    dec.conv_in = conv3("decoder.conv_in", ch[3], zc);
    dec.mid = stage("decoder.mid_block", {ch[3], ch[3]}, ch[3], 0, 0, 0, 1e-6f);
    vae_attn(dec, "decoder.mid_block.attentions.0", ch[3]);
    dec.blocks.clear();
    prev = ch[3];
    for (int i = 0; i < 4; ++i) {
      const int c = ch[3 - i];
      Stage s = stage("decoder.up_blocks." + std::to_string(i), {prev, c, c}, c, 0, 0, 0, 1e-6f);
      s.has_sampler = i < 3;
      if (s.has_sampler) s.sampler = upconv(s.name + ".upsamplers.0.conv", c, c);
      dec.blocks.push_back(std::move(s));
      prev = c;
    }
    dec.norm_out = norm("decoder.conv_norm_out", ch[0], 1e-6f);
    dec.conv_out = conv3("decoder.conv_out", cfg.out_channels, ch[0]);
  }

  // ---- CLIPVisionModelWithProjection (transformers key names)
  int clip_kpad() const { return static_cast<int>(rup(3LL * cfg.clip_patch_size * cfg.clip_patch_size, 64)); }
  void build_clip() {
    const int C = cfg.clip_hidden_size, heads = cfg.clip_heads, p = cfg.clip_patch_size, S = cfg.clip_image_size, I = cfg.clip_intermediate_size;
    const float eps = cfg.clip_layer_norm_eps;
    if (heads <= 0 || C != kClipHeadDim * heads) fail(HV_ERR_INVALID, "CLIP vision: hidden_size %d / %d heads: the head dim must be %d", C, heads, kClipHeadDim);
    if (C > 1280) fail(HV_ERR_INVALID, "CLIP vision: hidden_size %d is above the 1280 the LayerNorm kernel holds per row", C);
    if (p <= 0 || S <= 0 || S % p) fail(HV_ERR_INVALID, "CLIP vision: image_size %d must be a positive multiple of patch_size %d", S, p);
    if (cfg.clip_layers <= 0 || I <= 0 || I % 8 || cfg.clip_projection_dim <= 0 || !(eps > 0.f))
      fail(HV_ERR_INVALID, "CLIP vision: layers %d, intermediate_size %d (a multiple of 8), projection_dim %d and layer_norm_eps %g must be positive", cfg.clip_layers,
           I, cfg.clip_projection_dim, eps);
    const int L = (S / p) * (S / p) + 1;
    const std::string e = "vision_model.embeddings.";
    clip_patch = padded_linear(e + "patch_embedding", C, 3 * p * p, C, clip_kpad(), false);
    clip_cls = vec(e + "class_embedding", C);
    clip_pos = mat(e + "position_embedding.weight", L, C).p;
    clip_pre = norm("vision_model.pre_layrnorm", C, eps);
    clip_layers.clear();
    for (int i = 0; i < cfg.clip_layers; ++i) {
      const std::string pf = "vision_model.encoder.layers." + std::to_string(i) + ".";
      ClipLayerW w;
      w.ln1 = norm(pf + "layer_norm1", C, eps);
      w.ln2 = norm(pf + "layer_norm2", C, eps);
      const std::string a = pf + "self_attn.";
      w.attn = self_attn(a + "q_proj", a + "k_proj", a + "v_proj", a + "out_proj", C, heads, true);
      w.fc1 = lin(pf + "mlp.fc1", I, C);
      w.fc2 = lin(pf + "mlp.fc2", C, I);
      clip_layers.push_back(w);
    }
    clip_post = norm("vision_model.post_layernorm", C, eps);
    clip_proj = mat("visual_projection.weight", cfg.clip_projection_dim, C);
  }

  // ================================================================== op wrappers (no-ops while measuring)
  Tens alloc_act(int NF, int H, int W, int C) {
    Tens a;
    a.NF = NF; a.H = H; a.W = W; a.C = C;
    a.p = static_cast<__half*>(ar.alloc(static_cast<size_t>(a.numel()) * 2));
    return a;
  }
  __half* alloc_h(int64_t n) { return static_cast<__half*>(ar.alloc(static_cast<size_t>(n) * 2)); }

  // pool_F > 1: statistics over the pool_F frames of each batch item (same scratch; one finalize launch more)
  Tens op_gn(const Tens& x, const Tens* x2, const Norm& n, bool silu, int pool_F = 1) {
    const int C2 = x2 ? x2->C : 0;
    if (n.C != x.C + C2) fail(HV_ERR_INVALID, "groupnorm width %d != %d + %d", n.C, x.C, C2);
    Tens out = alloc_act(x.NF, x.H, x.W, x.C + C2);
    float* stats = static_cast<float*>(ar.alloc(sizeof(float) * groupnorm_scratch_floats(x.C + C2, x.NF, x.H * x.W, cfg.norm_groups)));
    if (pool_F > 1) {
      launch(3, {CAT_NORM, "groupnorm_pooled", 0, x.rows(), x.C + C2, 0}, [&] {   // statistics + finalize + apply
        ckop(op_groupnorm_pooled(x.p, x.C, x2 ? x2->p : nullptr, C2, n.g, n.b, out.p, x.NF, x.H * x.W, cfg.norm_groups, n.eps, silu ? 1 : 0, pool_F,
                                 stats, st),
             "groupnorm (pooled over frames)");
      });
      return out;
    }
    launch(2, {CAT_NORM, "groupnorm", 0, x.rows(), x.C + C2, 0}, [&] {   // statistics + apply
      ckop(op_groupnorm(x.p, x.C, x2 ? x2->p : nullptr, C2, n.g, n.b, out.p, x.NF, x.H * x.W, cfg.norm_groups, n.eps, silu ? 1 : 0, stats, st),
           "groupnorm");
    });
    return out;
  }
  // frames per batch item the resnet / conv_norm_out GroupNorms pool their statistics over (use_inflated_groupnorm=False); 1 = per frame
  int gn_pool(int F) const { return (cfg.kind == HV_KIND_UNET3D && cfg.gn_pool_frames) ? F : 1; }
  // (B, C, F, H, W) -> channels-last (B * F, H, W, Cpad), channels C .. Cpad zero (an input read as one 64-wide k-block)
  Tens padded_input(const __half* x, int B, int C, int F, int H, int W, int Cpad) {
    Tens t = alloc_act(B * F, H, W, Cpad);
    launch(2, {}, [&] {
      ck(cudaMemsetAsync(t.p, 0, static_cast<size_t>(t.numel()) * 2, st), "memset");
      ckop(op_ncfhw_to_nhwc(x, t.p, B, C, F, H, W, 0, st, Cpad), "input layout");
    });
    return t;
  }
  // out = LN(x (+ pre_add per batch item)) (+ pe per frame)
  Tens op_ln(const Tens& x, const Norm& n, const __half* pre_add = nullptr, int64_t rows_per_b = 1, const __half* pe = nullptr, int F = 1) {
    Tens out = alloc_act(x.NF, x.H, x.W, x.C);
    launch(1, {CAT_NORM, "layernorm", 0, x.rows(), x.C, 0}, [&] {
      ckop(op_layernorm(x.p, n.g, n.b, out.p, x.rows(), x.C, n.eps, pre_add, rows_per_b, nullptr, pe, x.H * x.W, F, st), "layernorm");
    });
    return out;
  }

  // out = e4m3(LN(x (+ pre_add per batch item)) (+ pe per frame)), one scale per row
  Q8 op_ln8(const Tens& x, const Norm& n, const __half* pre_add = nullptr, int64_t rows_per_b = 1, const __half* pe = nullptr, int F = 1) {
    Q8 out;
    out.t = x;
    out.t.p = nullptr;
    out.q = static_cast<uint8_t*>(ar.alloc(static_cast<size_t>(x.numel())));
    out.s = static_cast<float*>(ar.alloc(sizeof(float) * x.rows()));
    launch(1, {CAT_NORM, "layernorm_fp8", 0, x.rows(), x.C, 0}, [&] {
      ckop(op_layernorm_fp8(x.p, n.g, n.b, out.q, out.s, x.rows(), x.C, n.eps, pre_add, rows_per_b, nullptr, pe, x.H * x.W, F, st), "layernorm fp8");
    });
    return out;
  }
  // e4m3 linear of an e4m3 activation: fp16 out (+ bias, + rowvec[row / rows_per_group], + res), or, for a GEGLU-packed weight, e4m3 out
  // with one scale per 128 columns (the A operand of the next e4m3 linear)
  Tens op_linear8(const Q8& x, const Lin& l, const Tens* res = nullptr, const __half* rowvec = nullptr, int64_t rows_per_group = 1) {
    if (l.geglu) fail(HV_ERR_INVALID, "e4m3 linear with fp16 output: the weight is GEGLU-packed");
    return std::get<0>(run_linear8(x, l, res, rowvec, rows_per_group));
  }
  Q8 op_geglu8(const Q8& x, const Lin& l) {
    if (!l.geglu) fail(HV_ERR_INVALID, "e4m3 GEGLU: the weight is not GEGLU-packed");
    return std::get<1>(run_linear8(x, l, nullptr, nullptr, 1));
  }
  std::tuple<Tens, Q8> run_linear8(const Q8& x, const Lin& l, const Tens* res, const __half* rowvec, int64_t rows_per_group) {
    if (!l.w8) fail(HV_ERR_INVALID, "e4m3 linear: the weight has no e4m3 copy");
    if (l.w.cols != x.t.C) fail(HV_ERR_INVALID, "e4m3 linear: input width %d != weight cols %lld", x.t.C, (long long)l.w.cols);
    const int N = static_cast<int>(l.geglu ? l.w.rows / 2 : l.w.rows);
    Tens out;
    Q8 out8;
    if (l.geglu) {
      out8.t = x.t;
      out8.t.C = N;
      out8.t.p = nullptr;
      out8.sld = N / 128;
      out8.q = static_cast<uint8_t*>(ar.alloc(static_cast<size_t>(out8.t.numel())));
      out8.s = static_cast<float*>(ar.alloc(sizeof(float) * out8.t.rows() * out8.sld));
    } else {
      out = alloc_act(x.t.NF, x.t.H, x.t.W, N);
    }
    hv_epilogue ep = epilogue(l.bias, res, HV_ACT_NONE, rowvec, rows_per_group, N);
    ep.geglu = l.geglu ? 1 : 0;
    launch(1, {CAT_GEMM, l.geglu ? "gemm_geglu_fp8" : "gemm_fp8", 2.0 * x.t.rows() * l.w.rows * l.w.cols, x.t.rows(), l.w.rows, l.w.cols}, [&] {
      ckop(op_gemm_fp8(x.q, x.t.C, x.s, x.sld, l.w8, l.sw, l.geglu ? static_cast<void*>(out8.q) : static_cast<void*>(out.p), l.geglu ? N : out.C,
                       l.geglu ? out8.s : nullptr, out8.sld, x.t.rows(), l.w.rows, l.w.cols, &ep, st),
           "gemm fp8");
    });
    return {out, out8};
  }

  // The GEMM / conv wrappers write into `dst` (a tensor of the output's shape allocated by the caller) or into a new tensor.  Their
  // epilogue: + bias, + rowvec[row / rows_per_group] (rows of the output's width), act, + res.
  Tens dest(const Tens* dst, int NF, int H, int W, int C) {
    if (!dst) return alloc_act(NF, H, W, C);
    if (dst->NF != NF || dst->H != H || dst->W != W || dst->C != C)
      fail(HV_ERR_INVALID, "destination is (%d, %d, %d, %d), the output (%d, %d, %d, %d)", dst->NF, dst->H, dst->W, dst->C, NF, H, W, C);
    return *dst;
  }
  static hv_epilogue epilogue(const __half* bias, const Tens* res, int act, const __half* rowvec, int64_t rows_per_group, int N) {
    hv_epilogue e{};
    e.bias = bias;
    e.rowvec = rowvec;
    e.rowvec_ld = N;
    e.rows_per_group = static_cast<int32_t>(rows_per_group);
    e.act = act;
    if (res) { e.residual = res->p; e.ldr = res->C; }
    return e;
  }
  // out = [x | x2] W^T + epilogue; x2: a second source concatenated along K (the skip tensor of a resnet shortcut)
  Tens op_linear(const Tens& x, const Lin& l, const Tens* res = nullptr, const Tens* dst = nullptr, int act = HV_ACT_NONE, const Tens* x2 = nullptr,
                 const __half* rowvec = nullptr, int64_t rows_per_group = 1) {
    const int K1 = x2 ? x.C : 0, N = static_cast<int>(l.geglu ? l.w.rows / 2 : l.w.rows);
    if (l.w.cols != x.C + (x2 ? x2->C : 0)) fail(HV_ERR_INVALID, "linear: input width %d + %d != weight cols %lld", x.C, x2 ? x2->C : 0, (long long)l.w.cols);
    Tens out = dest(dst, x.NF, x.H, x.W, N);
    hv_epilogue ep = epilogue(l.bias, res, act, rowvec, rows_per_group, N);
    ep.geglu = l.geglu ? 1 : 0;
    launch(1, {CAT_GEMM, l.geglu ? "gemm_geglu" : (res ? "gemm_res" : "gemm"), 2.0 * x.rows() * l.w.rows * l.w.cols, x.rows(), l.w.rows, l.w.cols}, [&] {
      ckop(op_gemm(x.p, x.C, x2 ? x2->p : nullptr, x2 ? x2->C : 0, K1, l.w.p, out.p, out.C, x.rows(), l.w.rows, l.w.cols, &ep, st), "gemm");
    });
    return out;
  }
  // pad_end: stride 2 with padding (0, 1, 0, 1) (AutoencoderKL's Downsample2D) instead of 1 on every side
  Tens op_conv3(const Tens& x, const Conv3& c, int stride = 1, const Tens* res = nullptr, const Tens* dst = nullptr, int act = HV_ACT_NONE,
                const __half* rowvec = nullptr, int64_t rows_per_group = 1, bool pad_end = false) {
    if (x.C != c.cin_pad) fail(HV_ERR_INVALID, "conv3x3: input has %d channels, weight packed for %d", x.C, c.cin_pad);
    const int Ho = stride == 1 ? x.H : x.H / 2, Wo = stride == 1 ? x.W : x.W / 2;
    Tens out = dest(dst, x.NF, Ho, Wo, c.cout_pad);
    const hv_epilogue ep = epilogue(c.bias, res, act, rowvec, rows_per_group, c.cout_pad);
    const char* label = stride == 1 ? (res ? "conv3_res" : "conv3") : (pad_end ? "conv3_s2_end" : "conv3_s2");
    launch(1, {CAT_CONV, label, 2.0 * out.rows() * c.cout * 9.0 * c.cin, out.rows(), c.cout_pad, 9LL * c.cin_pad},
           [&] { ckop(op_conv3x3(x.p, c.w.p, out.p, out.C, x.NF, x.H, x.W, c.cin_pad, c.cout_pad, stride, &ep, st, pad_end), "conv3x3"); });
    return out;
  }
  // Upsample3D / Upsample2D: nearest 2x + 3x3 conv as four 2x2 convs of the source -- the 4x tensor is never materialised
  Tens op_upconv(const Tens& h, const Conv3& c, const Tens* dst = nullptr) {
    Tens big = dest(dst, h.NF, 2 * h.H, 2 * h.W, c.cout);
    const hv_epilogue ep = epilogue(c.bias, nullptr, HV_ACT_NONE, nullptr, 1, c.cout);
    launch(1, {CAT_CONV, "upconv2x2", 2.0 * big.rows() * c.cout * 4.0 * c.cin, big.rows(), c.cout, 4LL * c.cin},
           [&] { ckop(op_upconv2x2(h.p, c.w.p, big.p, big.C, h.NF, h.H, h.W, c.cin, c.cout, &ep, st), "upsampler conv"); });
    return big;
  }
  __half* op_small_linear(const __half* x, const Lin& l, int M, int act_in) {
    __half* out = alloc_h(static_cast<int64_t>(M) * l.w.rows);
    launch(1, {CAT_MISC, "", 2.0 * M * l.w.rows * l.w.cols}, [&] {
      ckop(hv::op_small_linear(x, l.w.p, l.bias, out, M, l.w.rows, l.w.cols, act_in, st), "small_linear");
    });
    return out;
  }

  // ================================================================== blocks
  // ResnetBlock3D (resnet.py:215-245); x2 = skip tensor concatenated on the channel axis (never materialised raw)
  Tens resnet_fwd(const ResnetW& r, const Tens& x, const Tens* x2, const __half* emb, int B, int F) {
    Tens out;
    {
      const int Cin = x.C + (x2 ? x2->C : 0);
      if (Cin != r.cin) fail(HV_ERR_INVALID, "resnet expects %d channels, got %d", r.cin, Cin);
      out = alloc_act(x.NF, x.H, x.W, r.cout);
    }
    Scope s(ar);
    __half* tproj = r.has_temb ? op_small_linear(emb, r.temb, B, HV_ACT_SILU) : nullptr;  // time_emb_proj(silu(emb)) : [B][cout]
    Tens h = op_gn(x, x2, r.n1, true, gn_pool(F));
    Tens h1 = op_conv3(h, r.c1, 1, nullptr, nullptr, HV_ACT_NONE, tproj, static_cast<int64_t>(F) * x.H * x.W);
    Tens h2 = op_gn(h1, nullptr, r.n2, true, gn_pool(F));
    Tens res = x;
    if (r.has_sc) res = op_linear(x, r.sc, nullptr, nullptr, HV_ACT_NONE, x2);
    else if (x2) fail(HV_ERR_INVALID, "resnet with concatenated input must have a shortcut conv");
    return op_conv3(h2, r.c2, 1, &res, &out);
  }

  // The reference bank a self-attention reads besides each frame's own tokens: keys [B][L][heads * dpad] and V^T with item i's tokens at
  // columns i * vt_stride; frame n reads item n / F, the first nf_nobank frames read none.
  struct BankKV {
    const __half* k = nullptr;
    const __half* vt = nullptr;
    int L = 0, F = 1, nf_nobank = 0;
    int64_t ldvt = 0, vt_stride = 0;
  };
  // Self-attention over each frame's H * W tokens of the normalised input xn: [Q | K] GEMM, V^T GEMM (frames side by side, its row bias
  // the ones rows and v's bias), the attention kernel, out = to_out(.) + bias + res.  bank() runs between the V^T GEMM and the attention
  // and returns the reference bank to read (the UNet's read / write hooks), or none.  The temporaries live in the caller's Scope.
  template <class BankFn>
  void self_attn_fwd(const SelfAttnW& a, const Tens& xn, const Tens& res, const Tens& out, BankFn&& bank) {
    const int C = xn.C, L = xn.H * xn.W;
    const int64_t hp = static_cast<int64_t>(a.heads) * a.dpad, Lp = rup(L, 8), ldvt = static_cast<int64_t>(xn.NF) * Lp;
    const int64_t vrows = a.wv.rows;
    Tens qk = op_linear(xn, a.qk);
    __half* vt = alloc_h(vrows * ldvt);
    // V^T[heads * dv][frame n: n * Lp + j] = Wv * xn^T: the weights are the "A" operand, the activations the batched "B" operand
    launch(1, {CAT_GEMM, "gemm_vt", 2.0 * xn.rows() * C * C, vrows, xn.rows(), C},
           [&] { ckop(op_gemm_batched_b(a.wv.p, C, xn.p, C, vt, ldvt, vrows, xn.NF, L, Lp, C, a.vbias, st), "V^T gemm"); });
    const BankKV b = bank();
    Tens o = alloc_act(xn.NF, xn.H, xn.W, C);
    const double flops = 4.0 * L * a.heads * a.d * (static_cast<double>(xn.NF) * L + static_cast<double>(xn.NF - b.nf_nobank) * b.L);
    if (a.dv == a.d) {   // single head, d = 512
      if (b.L > 0) fail(HV_ERR_INVALID, "the d = 512 attention reads no reference bank");
      launch(1, {CAT_ATTN, "attn_d512", flops, xn.NF, L, a.d},
             [&] { ckop(op_attention_d512(qk.p, 2 * hp, qk.p + hp, 2 * hp, vt, ldvt, Lp, o.p, C, xn.NF, L, st), "attention d512"); });
    } else {
      launch(1, {CAT_ATTN, "attn", flops, xn.NF, L, a.d}, [&] {
        ckop(op_attention(qk.p, qk.p + hp, vt, o.p, xn.NF, L, a.heads, a.d, 2 * hp, 2 * hp, ldvt, C, b.k, b.vt, b.L, hp, b.ldvt, b.F, b.nf_nobank, Lp,
                          b.vt_stride, st),
             "attention");
      });
    }
    op_linear(o, a.out, &res, &out);
  }

  // Transformer3DModel + TemporalBasicTransformerBlock (+ reference-bank read hook)
  Tens spatial_fwd(const SpatialW& w, const Tens& x, const __half* ehs, int B, int F, uint32_t flags) {
    Tens out = alloc_act(x.NF, x.H, x.W, x.C);
    Scope s(ar);
    const int C = w.C, L = x.H * x.W;
    Tens hn = op_gn(x, nullptr, w.gn, false);
    Tens t = op_linear(hn, w.proj_in);
    // ---- attn1
    Tens t1 = alloc_act(x.NF, x.H, x.W, C);  // t after self-attention residual
    {
      Scope s2(ar);
      Tens n1 = op_ln(t, w.ln1);
      self_attn_fwd(w.attn1, n1, t, t1, [&] {
        BankKV b;
        // write hook (mutual_self_attention.py:137-146): the bank IS LayerNorm-1's output; attention then runs on itself only
        if (bank_out != nullptr) {
          launch(1, {}, [&] {
            ck(cudaMemcpyAsync(bank_out[w.reader_idx], n1.p, static_cast<size_t>(n1.numel()) * 2, cudaMemcpyDeviceToDevice, st), "bank write");
          });
        }
        // HV_FLAG_CFG: batch = [uncond ; cond], the first half ignores the bank.  HV_FLAG_UNCOND_ONLY / HV_FLAG_COND_ONLY: the batch
        // holds one CFG half only (a (window x CFG-half) unit of a multi-GPU split); a cond-only batch of B items reads the LAST B
        // items of the bank (the bank is written for [uncond ; cond]).
        const bool cfg_split = (flags & HV_FLAG_CFG) != 0 && B >= 2 && B % 2 == 0 && !(flags & (HV_FLAG_UNCOND_ONLY | HV_FLAG_COND_ONLY));
        if (w.bank == nullptr || bank_out != nullptr || (flags & HV_FLAG_UNCOND_ONLY)) return b;
        int64_t item0 = 0;
        if (flags & HV_FLAG_COND_ONLY) {
          if (w.bank_B < B) fail(HV_ERR_INVALID, "reference bank of '%s' has batch %lld < forward batch %d", w.name.c_str(), (long long)w.bank_B, B);
          item0 = w.bank_B - B;
        } else if (w.bank_B != B && !ar.dry) {   // (a planning pass only sizes the workspace; it does not know the flags of the forward to come)
          fail(HV_ERR_INVALID, "reference bank of '%s' has batch %lld, forward batch is %d", w.name.c_str(), (long long)w.bank_B, B);
        }
        const SelfAttnW& a = w.attn1;
        const int64_t hp = static_cast<int64_t>(a.heads) * a.dpad;
        const Tens bank{w.bank + item0 * w.bank_L * C, B, 1, static_cast<int>(w.bank_L), C};
        b.k = op_linear(bank, Lin{Mat{a.qk.w.p + hp * C, hp, C}}).p;   // the K rows of [Q | K] (the UNet's projections have no bias)
        b.L = static_cast<int>(w.bank_L);
        b.F = F;
        b.nf_nobank = cfg_split ? (B / 2) * F : 0;
        b.vt_stride = rup(w.bank_L, 8);
        b.ldvt = static_cast<int64_t>(B) * b.vt_stride;
        __half* vbt = alloc_h(a.wv.rows * b.ldvt);
        b.vt = vbt;
        // its profile row has no label and no shape, so bench.py's per-shape GEMM roofline (gemm_classes) leaves it out
        launch(1, {CAT_GEMM, "", 2.0 * bank.rows() * C * C}, [&] {
          ckop(op_gemm_batched_b(a.wv.p, C, bank.p, C, vbt, b.ldvt, a.wv.rows, B, w.bank_L, b.vt_stride, C, a.vbias, st), "bank V^T gemm");
        });
        return b;
      });
    }
    // ---- attn2 with a single key: softmax == 1 -> out = to_out(to_v(ehs_b)) for every token of batch item b
    __half* v2 = op_small_linear(ehs, w.v2, B, HV_ACT_NONE);
    __half* ca = op_small_linear(v2, w.out2, B, HV_ACT_NONE);
    // LayerNorm-3 normalises t2 = t1 + ca[b] without writing t2: the same per-batch vector is added again, in fp32, in FF2's epilogue
    // (t3 = ff2(.) + bias + ca[b] + t1), which saves one full-tensor write per block and one rounding of the residual stream
    // ---- feed-forward, proj_out + residual
    Tens t3 = ff_fwd(t1, w.ln3, w.ff1, w.ff2, ca, static_cast<int64_t>(F) * L);
    return op_linear(t3, w.proj_out, &x, &out);
  }

  // one temporal attention sub-block: t = to_out(attn(LN(t) + pe)) + t
  Tens tattn_fwd(const TAttnW& a, const Tens& t, int B, int F, int heads, int d) {
    if (F > a.max_len) fail(HV_ERR_INVALID, "video_length %d exceeds temporal_position_encoding_max_len %d", F, a.max_len);
    Tens out = alloc_act(t.NF, t.H, t.W, t.C);
    Scope s(ar);
    const int C = t.C;
    Tens n = op_ln(t, a.ln, nullptr, 1, a.pe, F);
    Tens qkv = op_linear(n, a.qkv);
    Tens o = alloc_act(t.NF, t.H, t.W, C);
    launch(1, {CAT_TATTN, "tattn", 4.0 * t.rows() * F * C, t.rows(), F, C},
           [&] { ckop(op_temporal_attention(qkv.p, o.p, B, F, t.H * t.W, heads, d, st), "temporal attention"); });
    return op_linear(o, a.out, &t, &out);
  }
  // TemporalTransformerBlock: the temporal attentions, then t = ff(LN(t)) + t
  Tens tblock_fwd(const TBlockW& b, Tens t, int B, int F) {
    for (const auto& a : b.attn) t = tattn_fwd(a, t, B, F, b.heads, b.d);
    return ff_fwd(t, b.ff_norm, b.ff1, b.ff2);
  }
  // x + ff2(GEGLU ff1(LN(x + pre_add[b]))) + pre_add[b] (pre_add per batch item of rows_per_b rows, or none): on e4m3 when the weights carry
  // an e4m3 copy (fp8_ff), with the LayerNorm and GEGLU writing e4m3 and their scales
  Tens ff_fwd(const Tens& x, const Norm& n, const Lin& ff1, const Lin& ff2, const __half* pre_add = nullptr, int64_t rows_per_b = 1) {
    if (ff1.w8) return op_linear8(op_geglu8(op_ln8(x, n, pre_add, rows_per_b), ff1), ff2, &x, pre_add, rows_per_b);
    Tens ffh = op_linear(op_ln(x, n, pre_add, rows_per_b), ff1);
    return op_linear(ffh, ff2, &x, nullptr, HV_ACT_NONE, nullptr, pre_add, rows_per_b);
  }

  // VanillaTemporalModule (motion_module.py:44-259)
  Tens motion_fwd(const MotionW& m, const Tens& x, int B, int F) {
    Tens out = alloc_act(x.NF, x.H, x.W, x.C);
    Scope s(ar);
    Tens hn = op_gn(x, nullptr, m.gn, false);
    Tens t = op_linear(hn, m.proj_in);
    Tens t2 = tblock_fwd(m.block, t, B, F);
    return op_linear(t2, m.proj_out, &x, &out);
  }

  // ================================================================== forwards
  void begin(void* ws, size_t ws_bytes, bool dry, cudaStream_t stream) {
    st = stream;
    ar.dry = dry;
    ar.off = 0;
    ar.peak = 0;
    if (dry) {
      tap_list.clear();
      ar.base = nullptr;
      ar.cap = 0;
    } else {   // a planning pass keeps the launch count and the profile of the last forward
      ar.base = static_cast<uint8_t*>(ws);
      ar.cap = ws_bytes;
      launches = 0;
      recs.clear();
      ev_used = 0;
    }
  }

  void unet_forward(const __half* sample, int64_t timestep, const __half* ehs, const __half* pose, __half* outp, int B, int F, int H, int W,
                    uint32_t flags) {
    const int* ch = cfg.block_out_channels;
    const int NF = B * F;
    if ((H % 8) || (W % 8)) fail(HV_ERR_INVALID, "latent size %dx%d must be a multiple of 8 (three stride-2 levels)", H, W);
    // time embedding (unet_3d.py:446-467)
    __half* tsin = alloc_h(static_cast<int64_t>(B) * ch[0]);
    launch(1, {}, [&] { ckop(op_timestep_embedding(timestep, ts_table, ts_index, tsin, B, ch[0], st), "timestep embedding"); });
    __half* e1 = op_small_linear(tsin, te1, B, HV_ACT_NONE);
    __half* emb = op_small_linear(e1, te2, B, HV_ACT_SILU);
    // conv_in (+ pose_cond_fea as the epilogue residual)
    Tens x0 = padded_input(sample, B, cfg.in_channels, F, H, W, conv_in.cin_pad);
    Tens pc = pose ? alloc_act(NF, H, W, ch[0]) : Tens{};
    if (pose) launch(1, {}, [&] { ckop(op_ncfhw_to_nhwc(pose, pc.p, B, ch[0], F, H, W, 0, st), "pose layout"); });
    Tens h = op_conv3(x0, conv_in, 1, pose ? &pc : nullptr);
    tap("conv_in", h);
    // layer j of stage s (skip: the down-path tensor an up-path resnet concatenates)
    auto layer = [&](const Stage& s, size_t j, const Tens* skip) {
      const std::string sj = "." + std::to_string(j);
      h = resnet_fwd(s.res[j], h, skip, emb, B, F);
      tap(s.name + ".resnets" + sj, h);
      if (j < s.attn.size()) { h = spatial_fwd(s.attn[j], h, ehs, B, F, flags); tap(s.name + ".attentions" + sj, h); }
      if (j < s.mm.size()) { h = motion_fwd(s.mm[j], h, B, F); tap(s.name + ".motion_modules" + sj, h); }
    };
    std::vector<Tens> skips{h};
    for (const Stage& s : down) {
      for (size_t j = 0; j < s.res.size(); ++j) {
        layer(s, j, nullptr);
        skips.push_back(h);
      }
      if (s.has_sampler) {
        h = op_conv3(h, s.sampler, 2);
        tap(s.name + ".downsamplers.0", h);
        skips.push_back(h);
      }
    }
    layer(mid, 0, nullptr);
    layer(mid, 1, nullptr);
    for (const Stage& s : up) {
      for (size_t j = 0; j < s.res.size(); ++j) {
        const Tens skip = skips.back();
        skips.pop_back();
        layer(s, j, &skip);
      }
      if (s.has_sampler) {
        h = op_upconv(h, s.sampler);   // Upsample3D (resnet.py:68-71)
        tap(s.name + ".upsamplers.0", h);
      }
    }
    if (cfg.kind == HV_KIND_UNET2D_REF) {   // no post-process: the forward's value is the last up block's output (B, C0, h, w)
      if (outp != nullptr) launch(1, {}, [&] { ckop(op_nhwc_to_ncfhw(h.p, h.C, outp, B, ch[0], F, H, W, st), "hidden layout"); });
      return;
    }
    Tens hn = op_gn(h, nullptr, norm_out, true, gn_pool(F));
    Tens y = op_conv3(hn, conv_out);
    launch(1, {}, [&] { ckop(op_nhwc_to_ncfhw(y.p, y.C, outp, B, cfg.out_channels, F, H, W, st), "output layout"); });
  }

  void pose_guider_forward(const __half* cond, __half* outp, int B, int F, int H, int W) {
    const int NF = B * F;
    if ((H % 8) || (W % 8)) fail(HV_ERR_INVALID, "pose image %dx%d must be a multiple of 8", H, W);
    Tens h;
    if (pg_fast_in) {
      // conv_in (3 -> 16) straight from the (B, 3, F, H, W) image: no layout pass, 16-channel output
      h = alloc_act(NF, H, W, pg_in.cout);
      launch(1, {CAT_CONV, "pg_conv_in", 2.0 * h.rows() * pg_in.cout * 9.0 * pg_in.cin, h.rows(), pg_in.cout, 9LL * pg_in.cin},
             [&] { ckop(op_pose_conv_in(cond, pg_in.w, pg_in.bias, h.p, B, F, H, W, HV_ACT_SILU, st), "pose conv_in"); });
    } else {
      Tens x0 = alloc_act(NF, H, W, cfg.pg_cond_channels);
      h = alloc_act(NF, H, W, pg_convs[0].cin_pad);
      launch(3, {}, [&] {
        ckop(op_ncfhw_to_nhwc(cond, x0.p, B, cfg.pg_cond_channels, F, H, W, 0, st), "pose image layout");
        ck(cudaMemsetAsync(h.p, 0, static_cast<size_t>(h.numel()) * 2, st), "memset");
        ckop(op_conv3x3_direct(x0.p, pg_in.w, pg_in.bias, h.p, NF, H, W, pg_in.cin, pg_in.cout, 1, HV_ACT_SILU, nullptr, h.C, st), "pose conv_in");
      });
    }
    tap("conv_in", h);
    for (size_t i = 0; i < pg_convs.size(); ++i) {
      const bool last = i + 1 == pg_convs.size();
      const Conv3& c = pg_convs[i];
      const std::string name = last ? "conv_out" : "blocks." + std::to_string(i);
      if (pg_small[i]) {
        // the next layer either is a small-channel layer too (dense channels) or the first implicit-GEMM layer (its 64-multiple k-blocks)
        const int ld = pg_small[i + 1] ? c.cout : pg_convs[i + 1].cin_pad;
        const int Ho = pg_strides[i] == 1 ? h.H : h.H / 2, Wo = pg_strides[i] == 1 ? h.W : h.W / 2;
        if (h.C != c.cin) fail(HV_ERR_INVALID, "pose guider small conv %zu: input has %d channels, expects %d", i, h.C, c.cin);
        Tens out = alloc_act(NF, Ho, Wo, ld);
        if (ld > c.cout) launch(1, {}, [&] { ck(cudaMemsetAsync(out.p, 0, static_cast<size_t>(out.numel()) * 2, st), "memset"); });
        launch(1, {CAT_CONV, pg_strides[i] == 1 ? "smallconv" : "smallconv_s2", 2.0 * out.rows() * c.cout * 9.0 * c.cin, out.rows(), c.cout, 9LL * c.cin},
               [&] { ckop(op_conv3x3_small(h.p, c.w.p, c.bias, out.p, ld, NF, h.H, h.W, c.cin, c.cout, pg_strides[i], HV_ACT_SILU, st), "pose small conv"); });
        h = out;
        tap(name, h);
        continue;
      }
      h = op_conv3(h, c, pg_strides[i], nullptr, nullptr, last ? HV_ACT_NONE : HV_ACT_SILU);
      // the next conv expects cin_pad channels: cout_pad of this conv equals it by construction (both round to 64)
      if (!last && h.C != pg_convs[i + 1].cin_pad) fail(HV_ERR_INVALID, "pose guider channel padding mismatch at conv %zu", i);
      tap(name, h);
    }
    launch(1, {}, [&] { ckop(op_nhwc_to_ncfhw(h.p, h.C, outp, B, cfg.pg_out_channels, F, h.H, h.W, st), "pose output layout"); });
  }

  void camera_forward(const __half* plucker, __half* outp, int B, int F, int H, int W, const float* rays_K = nullptr, const float* rays_c2w = nullptr) {
    const int r = cfg.cam_downscale, NF = B * F, C = cfg.cam_channels;
    if ((H % r) || (W % r)) fail(HV_ERR_INVALID, "plucker map %dx%d must be a multiple of %d", H, W, r);
    const int cin0 = cfg.cam_cin / (r * r);
    Tens u = alloc_act(NF, H / r, W / r, cfg.cam_cin);
    if (rays_K != nullptr && cin0 != 6) fail(HV_ERR_INVALID, "the Plucker producer makes 6 channels, encoder expects %d", cin0);
    launch(1, {}, [&] {
      if (rays_K != nullptr)   // SURVEY 8f-3: Plucker embedding generated in place of the unshuffle's gather
        ckop(op_plucker_unshuffle(rays_K, rays_c2w, u.p, NF, H, W, r, st), "plucker unshuffle");
      else
        ckop(op_pixel_unshuffle(plucker, u.p, B, cin0, F, H, W, r, st), "pixel unshuffle");
    });
    Tens x = op_conv3(u, cam_in);
    tap("encoder_conv_in", x);
    for (int j = 0; j < cfg.cam_nums_rb; ++j) {
      const std::string sj = ".0." + std::to_string(j);
      // ResnetBlock (pose_adaptor.py:102-135, sk=True, ksize=1): x = block2(relu(block1(x))) + x
      Tens h1 = op_conv3(x, cam_res[j].block1, 1, nullptr, nullptr, HV_ACT_RELU);
      x = op_linear(h1, cam_res[j].block2, &x);
      tap("encoder_down_conv_blocks" + sj, x);
      x = tblock_fwd(cam_att[j], x, B, F);   // over the frame axis
      tap("encoder_down_attention_blocks" + sj, x);
    }
    Tens z = op_linear(x, cam_zero);
    tap("zero_conv_layers.0", z);
    launch(1, {}, [&] { ckop(op_nhwc_to_ncfhw(z.p, z.C, outp, NF, C, 1, z.H, z.W, st), "camera output layout"); });
  }

  // ================================================================== AutoencoderKL
  // UNetMidBlock2D: resnet, attention (diffusers Attention: GroupNorm, self-attention + residual), resnet
  Tens vae_mid_fwd(const VaeHalf& v, Tens h) {
    h = resnet_fwd(v.mid.res[0], h, nullptr, nullptr, h.NF, 1);
    tap(v.mid.name + ".resnets.0", h);
    Tens a = alloc_act(h.NF, h.H, h.W, h.C);
    {
      Scope s(ar);
      self_attn_fwd(v.attn, op_gn(h, nullptr, v.attn_gn, false), h, a, [] { return BankKV{}; });
    }
    tap(v.mid.name + ".attentions.0", a);
    h = resnet_fwd(v.mid.res[1], a, nullptr, nullptr, a.NF, 1);
    tap(v.mid.name + ".resnets.1", h);
    return h;
  }
  // the resnets and the sampler of one encoder / decoder stage
  Tens vae_stage_fwd(const Stage& s, Tens h, int N, bool down) {
    for (size_t j = 0; j < s.res.size(); ++j) {
      h = resnet_fwd(s.res[j], h, nullptr, nullptr, N, 1);
      tap(s.name + ".resnets." + std::to_string(j), h);
    }
    if (!s.has_sampler) return h;
    if (down) {
      h = op_conv3(h, s.sampler, 2, nullptr, nullptr, HV_ACT_NONE, nullptr, 1, true);   // Downsample2D: pad (0, 1, 0, 1), stride 2
      tap(s.name + ".downsamplers.0", h);
    } else {
      h = op_upconv(h, s.sampler);
      tap(s.name + ".upsamplers.0", h);
    }
    return h;
  }
  // Every operator works per frame (per-frame GroupNorm statistics, per-frame attention), so frame i of a call does not depend on the
  // other frames of the call.
  void vae_encode(const __half* x, __half* moments, int N, int H, int W) {
    if (N <= 0 || H <= 0 || W <= 0 || (H % 8) || (W % 8)) fail(HV_ERR_INVALID, "AutoencoderKL.encode: N = %d images of %dx%d: N must be > 0 and H, W positive multiples of 8", N, H, W);
    Tens x0 = padded_input(x, N, cfg.in_channels, 1, H, W, enc.conv_in.cin_pad);
    Tens h = op_conv3(x0, enc.conv_in);
    tap("encoder.conv_in", h);
    for (const Stage& s : enc.blocks) h = vae_stage_fwd(s, h, N, true);
    h = vae_mid_fwd(enc, h);
    Tens hn = op_gn(h, nullptr, enc.norm_out, true);
    tap("encoder.conv_norm_out", hn);
    Tens y = op_conv3(hn, enc.conv_out);
    tap("encoder.conv_out", y);
    Tens m = op_linear(y, quant);   // quant_conv (1x1)
    tap("quant_conv", m);
    launch(1, {}, [&] { ckop(op_nhwc_to_ncfhw(m.p, m.C, moments, N, m.C, 1, m.H, m.W, st), "moments layout"); });
  }
  void vae_decode(const __half* z, __half* outp, int N, int H, int W) {
    if (N <= 0 || H <= 0 || W <= 0) fail(HV_ERR_INVALID, "AutoencoderKL.decode: N = %d latents of %dx%d must all be positive", N, H, W);
    Tens z0 = padded_input(z, N, cfg.vae_latent_channels, 1, H, W, static_cast<int>(post_quant.w.cols));
    Tens p = op_linear(z0, post_quant);   // post_quant_conv (1x1); its padded channels stay zero for conv_in
    tap("post_quant_conv", p);
    Tens h = op_conv3(p, dec.conv_in);
    tap("decoder.conv_in", h);
    h = vae_mid_fwd(dec, h);
    for (const Stage& s : dec.blocks) h = vae_stage_fwd(s, h, N, false);
    Tens hn = op_gn(h, nullptr, dec.norm_out, true);
    tap("decoder.conv_norm_out", hn);
    Tens y = op_conv3(hn, dec.conv_out);
    tap("decoder.conv_out", y);
    launch(1, {}, [&] { ckop(op_nhwc_to_ncfhw(y.p, y.C, outp, N, cfg.out_channels, 1, y.H, y.W, st), "image output layout"); });
  }

  // ================================================================== CLIPVisionModelWithProjection
  // One CLIPEncoderLayer on the residual stream x ([B * L][hidden], image n's tokens in rows n L ..), result written to `out` (may be x):
  // LN1 -> [Q | K] (+bias) and V^T (+bias, ones rows) -> attention over each image's L tokens -> out_proj + bias + x -> LN2 -> fc1 + bias +
  // quick-GELU -> fc2 + bias + residual.
  void clip_layer_fwd(const ClipLayerW& w, const Tens& x, __half* out) {
    Scope s(ar);
    Tens n1 = op_ln(x, w.ln1);
    Tens h1 = alloc_act(x.NF, x.H, x.W, x.C);
    self_attn_fwd(w.attn, n1, x, h1, [] { return BankKV{}; });
    Tens n2 = op_ln(h1, w.ln2);
    Tens f = op_linear(n2, w.fc1, nullptr, nullptr, HV_ACT_QUICK_GELU);
    Tens y = x;
    y.p = out;
    op_linear(f, w.fc2, &h1, &y);
  }
  // pixels (B, 3, S, S) -> image_embeds (B, projection_dim) and, if lhs != nullptr, last_hidden_state (B, L, hidden).  Every operator works per
  // token row, per (image, head) or per output element, so image i of a call does not depend on the other images.
  void clip_forward(const __half* pix, __half* embeds, __half* lhs, int B, int S) {
    if (B <= 0 || S != cfg.clip_image_size)
      fail(HV_ERR_INVALID, "CLIPVisionModelWithProjection: %d images of %dx%d; the model takes a positive number of %dx%d images", B, S, S, cfg.clip_image_size,
           cfg.clip_image_size);
    const int C = cfg.clip_hidden_size, p = cfg.clip_patch_size, np = (S / p) * (S / p), L = np + 1, Kpad = clip_kpad();
    // patch embedding: the stride-p conv as patchify + GEMM
    Tens prow = alloc_act(B, 1, np, Kpad);
    launch(1, {}, [&] { ckop(op_clip_patchify(pix, prow.p, B, 3, S, p, Kpad, st), "patchify"); });
    Tens pe = op_linear(prow, clip_patch);
    // [class_embedding ; patches] + position_embedding -> pre_layrnorm: the residual stream (B images x L tokens)
    Tens x = alloc_act(B, 1, L, C);
    launch(1, {CAT_NORM, "clip_embed_ln", 0, x.rows(), C, 0},
           [&] { ckop(op_clip_embed_ln(pe.p, clip_cls, clip_pos, clip_pre.g, clip_pre.b, x.p, x.rows(), L, C, clip_pre.eps, st), "embeddings + pre_layrnorm"); });
    tap("vision_model.pre_layrnorm", x);
    for (size_t i = 0; i < clip_layers.size(); ++i) {
      const bool last = i + 1 == clip_layers.size();
      __half* dst = last && lhs != nullptr ? lhs : x.p;   // the stream is updated in place; the last layer writes the caller's last_hidden_state
      clip_layer_fwd(clip_layers[i], x, dst);
      x.p = dst;
      tap("vision_model.encoder.layers." + std::to_string(i), x);
    }
    // pooling: the class token of each image -> post_layernorm -> visual_projection (no bias)
    Tens cls = alloc_act(B, 1, 1, C);
    launch(1, {}, [&] {
      ck(cudaMemcpy2DAsync(cls.p, static_cast<size_t>(C) * 2, x.p, static_cast<size_t>(L) * C * 2, static_cast<size_t>(C) * 2, B, cudaMemcpyDeviceToDevice, st),
         "class tokens");
    });
    Tens pooled = op_ln(cls, clip_post);
    tap("vision_model.post_layernorm", pooled);
    const int P = static_cast<int>(clip_proj.rows);
    launch(1, {CAT_MISC, "", 2.0 * B * P * C},
           [&] { ckop(hv::op_small_linear(pooled.p, clip_proj.p, nullptr, embeds, B, P, C, HV_ACT_NONE, st), "visual_projection"); });
  }
};

// ------------------------------------------------------------------------------------------ C ABI
// Runs fn and turns an exception into its status; the message goes to hv_last_error(h) and to the library's last error.
template <class Fn>
static int guard(hv_model* h, Fn&& fn) {
  try {
    fn();
    return HV_OK;
  } catch (const Err& e) {
    if (h) h->err = e.msg;
    set_error("%s", e.msg.c_str());
    return e.code;
  } catch (const std::exception& e) {
    if (h) h->err = e.what();
    set_error("%s", e.what());
    return HV_ERR_INVALID;
  }
}

// The forwards never allocate: a caller that passes no workspace must have called hv_reserve_workspace for a shape at least as
// large (cudaMalloc synchronises the device and is illegal under stream capture).
static void* get_ws(hv_model* m, void* ws, size_t ws_bytes, size_t need, size_t* have) {
  if (ws) {
    *have = ws_bytes;
    return ws;
  }
  if (m->private_ws_bytes < need)
    fail(HV_ERR_STATE, "workspace == NULL and the handle's reserved workspace (%zu bytes) is smaller than the %zu this shape needs: call hv_reserve_workspace first",
         m->private_ws_bytes, need);
  *have = m->private_ws_bytes;
  return m->private_ws;
}

// The planning pass: returns the workspace one forward needs at this shape and leaves the plan of its taps in tap_list.
static size_t measure(hv_model* h, int B, int F, int H, int W, uint32_t flags = HV_FLAG_CFG) {
  h->begin(nullptr, 0, true, nullptr);
  if (h->cfg.kind == HV_KIND_UNET3D || h->cfg.kind == HV_KIND_UNET2D_REF) {
    static __half dummy;
    h->unet_forward(&dummy, 0, &dummy, h->cfg.kind == HV_KIND_UNET3D ? &dummy : nullptr, &dummy, B, F, H, W, flags);
  } else if (h->cfg.kind == HV_KIND_POSE_GUIDER) {
    h->pose_guider_forward(nullptr, nullptr, B, F, H, W);
  } else if (h->cfg.kind == HV_KIND_VAE) {   // (H, W) = latent size: the workspace covers decoding B latents and encoding B images of 8H x 8W
    h->vae_decode(nullptr, nullptr, B, H, W);
    const size_t dec_peak = h->ar.peak;
    h->ar.off = h->ar.peak = 0;   // the encode on an empty arena; its taps follow the decoder's in tap_list
    h->vae_encode(nullptr, nullptr, B, 8 * H, 8 * W);
    return std::max(dec_peak, h->ar.peak) + 4096;
  } else if (h->cfg.kind == HV_KIND_CLIP_VISION) {   // (B, 1, S, S): B images of S x S pixels
    if (F != 1 || H != W) fail(HV_ERR_INVALID, "CLIPVisionModelWithProjection: workspace shape (B, F, H, W) = (%d, %d, %d, %d) must be (B, 1, S, S)", B, F, H, W);
    h->clip_forward(nullptr, nullptr, nullptr, B, H);
  } else {
    h->camera_forward(nullptr, nullptr, B, F, H, W);
  }
  return h->ar.peak + 4096;
}

// Plans the forward at this shape, binds the workspace and the stream, and runs fwd.
template <class Fwd>
static void run_forward(hv_model* h, int kind, const char* what, int B, int F, int H, int W, uint32_t flags, void* workspace, size_t ws_bytes,
                        hv_stream_t stream, Fwd&& fwd) {
  if (!h->finalized || h->cfg.kind != kind) fail(HV_ERR_STATE, "handle is not a finalized %s", what);
  const size_t need = measure(h, B, F, H, W, flags);
  size_t have = 0;
  void* ws = get_ws(h, workspace, ws_bytes, need, &have);
  h->begin(ws, have, false, static_cast<cudaStream_t>(stream));
  fwd();
}

extern "C" {

int hv_create(const hv_config* cfg, hv_handle* out) {
  if (!cfg || !out) return HV_ERR_INVALID;
  hv_model* m = nullptr;
  try {
    if (!device_sms()) fail(HV_ERR_CUDA, "%s", last_error());
    m = new hv_model();
    m->cfg = *cfg;
    if (cfg->kind < 0 || cfg->kind > HV_KIND_CLIP_VISION) fail(HV_ERR_INVALID, "unknown kind %d", cfg->kind);
    if (cfg->kind == HV_KIND_UNET2D_REF && cfg->use_motion_module) fail(HV_ERR_INVALID, "the reference (writer) UNet has no motion modules");
    *out = m;
    return HV_OK;
  } catch (const Err& e) {
    set_error("%s", e.msg.c_str());
    delete m;
    return e.code;
  }
}

void hv_destroy(hv_handle h) { delete h; }
const char* hv_last_error(hv_handle h) { return h ? h->err.c_str() : last_error(); }
int64_t hv_last_launch_count(hv_handle h) { return h ? h->launches : 0; }

int hv_set_profiling(hv_handle h, int32_t enable) {
  if (!h) return HV_ERR_INVALID;
  h->profiling = enable != 0;
  return HV_OK;
}

int hv_dump_profile(hv_handle h, const char* path) {
  if (!h || !path) return HV_ERR_INVALID;
  return guard(h, [&] {
    FILE* f = fopen(path, "w");
    if (!f) fail(HV_ERR_INVALID, "cannot open %s", path);
    if (!h->recs.empty()) ck(cudaEventSynchronize(h->recs.back().b), "profile sync");
    fprintf(f, "idx,cat,label,M,N,K,ms,tflops\n");
    int i = 0;
    for (const auto& r : h->recs) {
      float t = 0;
      cudaEventElapsedTime(&t, r.a, r.b);
      fprintf(f, "%d,%d,%s,%lld,%lld,%lld,%.4f,%.1f\n", i++, r.cat, r.label, r.m, r.n, r.k, t, t > 0 ? r.flops / 1e9 / t : 0.0);
    }
    fclose(f);
  });
}

int hv_get_profile(hv_handle h, double* ms, double* flops, int64_t* count, int32_t ncat) {
  if (!h || !ms || !flops || !count) return HV_ERR_INVALID;
  return guard(h, [&] {
    for (int i = 0; i < ncat; ++i) { ms[i] = 0; flops[i] = 0; count[i] = 0; }
    if (!h->recs.empty()) ck(cudaEventSynchronize(h->recs.back().b), "profile sync");
    for (const auto& r : h->recs) {
      if (r.cat >= ncat) continue;
      float t = 0;
      ck(cudaEventElapsedTime(&t, r.a, r.b), "cudaEventElapsedTime");
      ms[r.cat] += t;
      flops[r.cat] += r.flops;
      count[r.cat] += 1;
    }
  });
}

__global__ void cast_f32_to_f16(const float* __restrict__ x, __half* __restrict__ y, long long n) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x)
    y[i] = __float2half_rn(x[i]);
}

int hv_set_weight(hv_handle h, const char* key, const void* dev_ptr, const int64_t* shape, int32_t ndim, int32_t dtype, hv_stream_t stream) {
  if (!h || !key || !dev_ptr || ndim < 0 || ndim > 8) return HV_ERR_INVALID;
  return guard(h, [&] {
    if (h->finalized) fail(HV_ERR_STATE, "hv_set_weight after hv_finalize");
    Raw r;
    r.shape.assign(shape, shape + ndim);
    const int64_t n = r.numel();
    if (n <= 0) fail(HV_ERR_INVALID, "weight '%s' is empty", key);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    void* p = nullptr;
    ck(cudaMalloc(&p, static_cast<size_t>(rup(n, 8)) * 2), "cudaMalloc(weight)");
    h->owned.push_back(p);
    r.p = static_cast<__half*>(p);
    if (dtype == HV_F16) {
      ck(cudaMemcpyAsync(r.p, dev_ptr, static_cast<size_t>(n) * 2, cudaMemcpyDeviceToDevice, st), "weight copy");
    } else if (dtype == HV_F32) {
      long long blocks = std::min<long long>((n + 255) / 256, 4096);
      cast_f32_to_f16<<<static_cast<unsigned>(blocks), 256, 0, st>>>(static_cast<const float*>(dev_ptr), r.p, n);
      ck(cudaGetLastError(), "weight cast");
    } else {
      fail(HV_ERR_INVALID, "weight '%s': unsupported dtype %d", key, dtype);
    }
    h->raw[key] = r;
  });
}

int hv_finalize(hv_handle h, hv_stream_t stream) {
  if (!h) return HV_ERR_INVALID;
  return guard(h, [&] {
    if (h->finalized) return;
    h->st = static_cast<cudaStream_t>(stream);
    if (h->cfg.kind == HV_KIND_UNET3D || h->cfg.kind == HV_KIND_UNET2D_REF) h->build_unet();
    else if (h->cfg.kind == HV_KIND_POSE_GUIDER) h->build_pose_guider();
    else if (h->cfg.kind == HV_KIND_VAE) h->build_vae();
    else if (h->cfg.kind == HV_KIND_CLIP_VISION) h->build_clip();
    else h->build_camera();
    h->finalized = true;
  });
}

int hv_num_ref_blocks(hv_handle h) { return (h && h->finalized) ? static_cast<int>(h->readers.size()) : 0; }
int hv_ref_block_dim(hv_handle h, int32_t i) {
  return (h && h->finalized && i >= 0 && i < static_cast<int>(h->readers.size())) ? h->readers[i]->C : 0;
}

int hv_set_ref_bank(hv_handle h, int32_t idx, const void* dev_ptr, int64_t B_ref, int64_t L, int64_t C, hv_stream_t stream) {
  if (!h) return HV_ERR_INVALID;
  return guard(h, [&] {
    if (!h->finalized) fail(HV_ERR_STATE, "hv_set_ref_bank before hv_finalize");
    if (idx < 0 || idx >= static_cast<int>(h->readers.size())) fail(HV_ERR_INVALID, "bank index %d out of range", idx);
    SpatialW* w = h->readers[idx];
    if (C != w->C) fail(HV_ERR_INVALID, "bank %d has width %lld, block '%s' has %d", idx, (long long)C, w->name.c_str(), w->C);
    const int64_t n = B_ref * L * C;
    if (w->bank_cap < n) {
      w->bank_store = h->dmalloc(n);
      w->bank_cap = n;
    }
    w->bank = w->bank_store;
    w->bank_B = B_ref;
    w->bank_L = L;
    ck(cudaMemcpyAsync(w->bank, dev_ptr, static_cast<size_t>(n) * 2, cudaMemcpyDeviceToDevice, static_cast<cudaStream_t>(stream)), "bank copy");
  });
}

int hv_clear_ref_banks(hv_handle h) {
  if (!h) return HV_ERR_INVALID;
  for (SpatialW* w : h->readers) {
    w->bank = nullptr;  // bank_store is kept for the next hv_set_ref_bank
    w->bank_B = w->bank_L = 0;
  }
  return HV_OK;
}

int hv_reserve_workspace(hv_handle h, int32_t B, int32_t F, int32_t height, int32_t width) {
  if (!h) return HV_ERR_INVALID;
  return guard(h, [&] {
    if (!h->finalized) fail(HV_ERR_STATE, "hv_reserve_workspace before hv_finalize");
    const size_t need = measure(h, B, F, height, width);
    if (h->private_ws_bytes < need) {
      if (h->private_ws) ck(cudaFree(h->private_ws), "cudaFree(workspace)");
      h->private_ws = nullptr;
      h->private_ws_bytes = 0;
      ck(cudaMalloc(&h->private_ws, need), "cudaMalloc(workspace)");
      h->private_ws_bytes = need;
    }
  });
}

int hv_set_timestep_source(hv_handle h, const int64_t* dev_table, const int32_t* dev_index) {
  if (!h || ((dev_table == nullptr) != (dev_index == nullptr))) return HV_ERR_INVALID;
  h->ts_table = reinterpret_cast<const long long*>(dev_table);
  h->ts_index = dev_index;
  return HV_OK;
}

int hv_debug_tap_count(hv_handle h, int32_t B, int32_t F, int32_t height, int32_t width) {
  if (!h || !h->finalized) return HV_ERR_INVALID;
  const int status = guard(h, [&] { measure(h, B, F, height, width); });
  return status == HV_OK ? static_cast<int>(h->tap_list.size()) : status;
}

int hv_debug_tap_info(hv_handle h, int32_t i, char* name, int32_t name_cap, int64_t* dims4) {
  if (!h || !name || !dims4 || i < 0 || i >= static_cast<int>(h->tap_list.size()) || name_cap <= 0) return HV_ERR_INVALID;
  const auto& t = h->tap_list[i];
  snprintf(name, static_cast<size_t>(name_cap), "%s", t.name.c_str());
  dims4[0] = t.NF; dims4[1] = t.H; dims4[2] = t.W; dims4[3] = t.C;
  return HV_OK;
}

int hv_debug_set_taps(hv_handle h, void* const* dst, int32_t n) {
  if (!h || n < 0 || (n > 0 && !dst)) return HV_ERR_INVALID;
  h->tap_dst.assign(dst, dst + n);
  return HV_OK;
}

size_t hv_workspace_bytes(hv_handle h, int32_t B, int32_t F, int32_t height, int32_t width) {
  if (!h || !h->finalized) return 0;
  size_t need = 0;
  return guard(h, [&] { need = measure(h, B, F, height, width); }) == HV_OK ? need : 0;
}

int hv_unet3d_forward(hv_handle h, const void* sample, int64_t timestep, const void* ehs, const void* pose, void* out, int32_t B, int32_t F,
                      int32_t height, int32_t width, uint32_t flags, void* workspace, size_t ws_bytes, hv_stream_t stream) {
  if (!h || !sample || !ehs || !out) return HV_ERR_INVALID;
  return guard(h, [&] {
    if ((flags & HV_FLAG_UNCOND_ONLY) && (flags & HV_FLAG_COND_ONLY)) fail(HV_ERR_INVALID, "HV_FLAG_UNCOND_ONLY and HV_FLAG_COND_ONLY are exclusive");
    run_forward(h, HV_KIND_UNET3D, "UNet3D", B, F, height, width, flags, workspace, ws_bytes, stream, [&] {
      h->unet_forward(static_cast<const __half*>(sample), timestep, static_cast<const __half*>(ehs), static_cast<const __half*>(pose),
                      static_cast<__half*>(out), B, F, height, width, flags);
    });
  });
}

int hv_unet2d_reference_forward(hv_handle h, const void* sample, int64_t timestep, const void* ehs, void* hidden_out, void* const* bank_out,
                                int32_t n_banks, int32_t B, int32_t height, int32_t width, void* workspace, size_t ws_bytes, hv_stream_t stream) {
  if (!h || !sample || !ehs || !bank_out) return HV_ERR_INVALID;
  return guard(h, [&] {
    run_forward(h, HV_KIND_UNET2D_REF, "reference (writer) UNet2D", B, 1, height, width, HV_FLAG_CFG, workspace, ws_bytes, stream, [&] {
      if (n_banks != static_cast<int>(h->readers.size())) fail(HV_ERR_INVALID, "expected %d bank destinations, got %d", (int)h->readers.size(), n_banks);
      for (int i = 0; i < n_banks; ++i)
        if (bank_out[i] == nullptr) fail(HV_ERR_INVALID, "bank destination %d is NULL", i);
      struct BankOut {   // the bank destinations belong to this forward only
        hv_model* m;
        ~BankOut() { m->bank_out = nullptr; }
      } reset{h};
      h->bank_out = reinterpret_cast<__half* const*>(bank_out);
      h->unet_forward(static_cast<const __half*>(sample), timestep, static_cast<const __half*>(ehs), nullptr, static_cast<__half*>(hidden_out), B, 1,
                      height, width, 0);
    });
  });
}

int hv_pose_guider_forward(hv_handle h, const void* cond, void* out, int32_t B, int32_t F, int32_t H, int32_t W, void* workspace,
                           size_t ws_bytes, hv_stream_t stream) {
  if (!h || !cond || !out) return HV_ERR_INVALID;
  return guard(h, [&] {
    run_forward(h, HV_KIND_POSE_GUIDER, "PoseGuider", B, F, H, W, HV_FLAG_CFG, workspace, ws_bytes, stream,
                [&] { h->pose_guider_forward(static_cast<const __half*>(cond), static_cast<__half*>(out), B, F, H, W); });
  });
}

int hv_camera_encoder_forward(hv_handle h, const void* plucker, void* out, int32_t B, int32_t F, int32_t H, int32_t W, void* workspace,
                              size_t ws_bytes, hv_stream_t stream) {
  if (!h || !plucker || !out) return HV_ERR_INVALID;
  return guard(h, [&] {
    run_forward(h, HV_KIND_CAMERA_ENCODER, "CameraPoseEncoder", B, F, H, W, HV_FLAG_CFG, workspace, ws_bytes, stream,
                [&] { h->camera_forward(static_cast<const __half*>(plucker), static_cast<__half*>(out), B, F, H, W); });
  });
}

int hv_camera_encoder_forward_rays(hv_handle h, const float* intrinsics, const float* c2w, void* out, int32_t B, int32_t F, int32_t H, int32_t W,
                                   void* workspace, size_t ws_bytes, hv_stream_t stream) {
  if (!h || !intrinsics || !c2w || !out) return HV_ERR_INVALID;
  return guard(h, [&] {
    run_forward(h, HV_KIND_CAMERA_ENCODER, "CameraPoseEncoder", B, F, H, W, HV_FLAG_CFG, workspace, ws_bytes, stream,
                [&] { h->camera_forward(nullptr, static_cast<__half*>(out), B, F, H, W, intrinsics, c2w); });
  });
}

int hv_vae_decode(hv_handle h, const void* z, void* out, int32_t N, int32_t height, int32_t width, void* workspace, size_t ws_bytes,
                  hv_stream_t stream) {
  if (!h || !z || !out) return HV_ERR_INVALID;
  return guard(h, [&] {
    run_forward(h, HV_KIND_VAE, "AutoencoderKL", N, 1, height, width, 0, workspace, ws_bytes, stream,
                [&] { h->vae_decode(static_cast<const __half*>(z), static_cast<__half*>(out), N, height, width); });
  });
}

int hv_vae_encode(hv_handle h, const void* x, void* moments, int32_t N, int32_t H, int32_t W, void* workspace, size_t ws_bytes,
                  hv_stream_t stream) {
  if (!h || !x || !moments) return HV_ERR_INVALID;
  return guard(h, [&] {
    if (N <= 0 || H <= 0 || W <= 0 || (H % 8) || (W % 8))
      fail(HV_ERR_INVALID, "AutoencoderKL.encode: N = %d images of %dx%d: N must be > 0 and H, W positive multiples of 8", N, H, W);
    run_forward(h, HV_KIND_VAE, "AutoencoderKL", N, 1, H / 8, W / 8, 0, workspace, ws_bytes, stream,
                [&] { h->vae_encode(static_cast<const __half*>(x), static_cast<__half*>(moments), N, H, W); });
  });
}

int hv_clip_vision_forward(hv_handle h, const void* pixel_values, void* image_embeds, void* last_hidden_state, int32_t B, void* workspace,
                           size_t ws_bytes, hv_stream_t stream) {
  if (!h || !pixel_values || !image_embeds) return HV_ERR_INVALID;
  return guard(h, [&] {
    const int S = h->cfg.clip_image_size;
    run_forward(h, HV_KIND_CLIP_VISION, "CLIPVisionModelWithProjection", B, 1, S, S, 0, workspace, ws_bytes, stream, [&] {
      h->clip_forward(static_cast<const __half*>(pixel_values), static_cast<__half*>(image_embeds), static_cast<__half*>(last_hidden_state), B, S);
    });
  });
}

}  // extern "C"
