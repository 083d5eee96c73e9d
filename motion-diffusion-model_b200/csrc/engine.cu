// libb200mdm.so -- C-ABI engine (see include/b200mdm.h for the contract and the reference lines each entry
// point replaces).  Host side: weight store + repack, TMA descriptor set-up, per-(B,T) workspace, launch
// sequences for one denoiser forward / one sampler step, and the whole-loop driver (one CUDA graph of a single
// step, replayed; per-step scalars are read from device tables indexed by a device-side step counter so the
// graph never changes).
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <initializer_list>
#include <map>
#include <string>
#include <vector>

#include "../../include/b200mdm.h"
#include "attention_tc.cuh"
#include "epilogues.cuh"
#include "gemm.cuh"
#include "gemm_ln.cuh"
#include "gemm_pingpong.cuh"
#include "chunk_frame.cuh"
#include "joint_guidance.cuh"
#include "compose.cuh"
#include "postprocess.cuh"
#include "kernels.cuh"

using namespace b200;

// ------------------------------------------------------------------------------------------------ errors
static thread_local char g_err[512] = "";
static int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}
#define CUDA_TRY(expr)                                                                               \
  do {                                                                                               \
    cudaError_t _e = (expr);                                                                         \
    if (_e != cudaSuccess)                                                                           \
      return fail(B200MDM_ECUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)
#define TRY(expr)            \
  do {                       \
    int _r = (expr);         \
    if (_r != B200MDM_OK) return _r; \
  } while (0)

// ------------------------------------------------------------------------------------------------ TMA maps
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn g_encode = nullptr;
static int resolve_driver() {
  if (g_encode) return B200MDM_OK;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  CUDA_TRY(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
  if (!fn || qres != cudaDriverEntryPointSuccess) return fail(B200MDM_ECUDA, "cuTensorMapEncodeTiled not available");
  g_encode = reinterpret_cast<EncodeTiledFn>(fn);
  return B200MDM_OK;
}
// One cuTensorMapEncodeTiled call: `rank` dimensions gdim (innermost first) with rank - 1 byte pitches, no interleave,
// 256-byte L2 promotion, out-of-bounds elements read as zero.
static int encode_map(CUtensorMap* m, CUtensorMapDataType dtype, uint32_t rank, const void* ptr, const cuuint64_t* gdim,
                      const cuuint64_t* gstride_bytes, const cuuint32_t* box, CUtensorMapSwizzle swizzle, const char* what) {
  TRY(resolve_driver());
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) || gstride_bytes[0] % 16) return fail(B200MDM_EINVAL, "TMA operand misaligned");
  const cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = g_encode(m, dtype, rank, const_cast<void*>(ptr), gdim, gstride_bytes, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(B200MDM_ECUDA, "cuTensorMapEncodeTiled%s failed (%d)", what, static_cast<int>(r));
  return B200MDM_OK;
}
// fp16 matrix [rows, cols] with leading dimension ld (elements); box = box_rows x 64 columns, 128-byte swizzle.
// elem_bytes 2 = fp16, 4 = fp32; the box is always 128 bytes wide (64 fp16 / 32 fp32 columns) x box_rows.
static int make_map_t(CUtensorMap* m, const void* ptr, int elem_bytes, uint64_t rows, uint64_t cols, uint64_t ld,
                      uint32_t box_rows) {
  const cuuint64_t gdim[2] = {cols, rows}, gstr[1] = {ld * elem_bytes};
  const cuuint32_t box[2] = {static_cast<cuuint32_t>(128 / elem_bytes), box_rows};
  return encode_map(m, elem_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, ptr, gdim, gstr,
                    box, CU_TENSOR_MAP_SWIZZLE_128B, "");
}
static int make_map(CUtensorMap* m, const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows) {
  return make_map_t(m, ptr, 2, rows, cols, ld, box_rows);
}
// fp16 tensor viewed [n][rows][cols] (cols contiguous, row pitch ld elements, sample pitch rows*ld); box {64, box_rows, 1}.
// The middle dimension is bounded per sample, so tiles that run past the last token of a sample are zero-filled.
static int make_map_3d(CUtensorMap* m, const void* ptr, uint64_t n, uint64_t rows, uint64_t cols, uint64_t ld,
                       uint32_t box_rows) {
  const cuuint64_t gdim[3] = {cols, rows, n}, gstr[2] = {ld * 2, rows * ld * 2};
  const cuuint32_t box[3] = {64, box_rows, 1};
  return encode_map(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, ptr, gdim, gstr, box, CU_TENSOR_MAP_SWIZZLE_128B, "(3d)");
}

// Residual stream [M, 2 x 512] fp16 as the residual + LayerNorm GEMM moves it: box 64 columns x GLN_RES_BOX_ROWS rows.
static int make_hres_map(CUtensorMap* m, const void* hres, uint64_t rows) {
  return make_map(m, hres, rows, 2 * GLN_D, 2 * GLN_D, GLN_RES_BOX_ROWS);
}

// Residual stream fp16 [rows, 2d] = [hi | lo]: box {32 cols, 32 rows} with 64-byte rows and the 64-byte swizzle; an
// epilogue chunk of 32 columns moves one such box from the hi half and one from the lo half.
static int make_map_res(CUtensorMap* m, const void* ptr, uint64_t rows, uint64_t d) {
  const cuuint64_t gdim[2] = {2 * d, rows}, gstr[1] = {d * 4};
  const cuuint32_t box[2] = {32, 32};
  return encode_map(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, ptr, gdim, gstr, box, CU_TENSOR_MAP_SWIZZLE_64B, "(residual)");
}

// ------------------------------------------------------------------------------------------------ engine
// The schedule's row tables, one row per schedule index: the step table (b200mdm_set_schedule), the DDIM inversion's
// sqrt(abn), sqrt(1 - abn), DPM-Solver++'s c_x, c0, c_cur, c_prev and the variational bound's VB_* columns.
enum SchedTable { TAB_STEP, TAB_NEXT, TAB_DPM, TAB_VB, N_TABLES };
static constexpr int TAB_STRIDE[N_TABLES] = {SCHED_STRIDE, SCHED_NEXT_STRIDE, SCHED_DPM_STRIDE, SCHED_VB_STRIDE};
static const char* const TAB_SETTER[N_TABLES] = {"b200mdm_set_schedule", "b200mdm_set_schedule_next",
                                                 "b200mdm_set_schedule_dpm", "b200mdm_set_schedule_vb"};
static_assert(SCHED_STRIDE == B200MDM_SCHED_STRIDE && SCHED_NEXT_STRIDE == B200MDM_SCHED_NEXT_STRIDE &&
                  SCHED_DPM_STRIDE == B200MDM_SCHED_DPM_STRIDE && SCHED_VB_STRIDE == B200MDM_SCHED_VB_STRIDE,
              "the tables' row layouts are part of the ABI");

struct Tensor32 {
  float* dev = nullptr;
  std::vector<int64_t> shape;
  size_t numel = 0;
};

struct LayerW {
  __half *wqkv = nullptr, *wo = nullptr, *w1 = nullptr, *w2 = nullptr;
  const float *bqkv, *bo, *b1, *b2, *g1, *be1, *g2, *be2;
  CUtensorMap m_wqkv, m_w1;               // box 128 rows: the 128-column W tiles of the projection GEMMs
  CUtensorMap m_wo_256, m_w2_256;         // box 256 rows: residual+LayerNorm kernel (each CTA owns 256 output columns)
  // trans_dec only: cross-attention (multihead_attn) projections and the third LayerNorm
  __half *wq_c = nullptr, *wo_c = nullptr;           // (the K/V rows of all layers live in engine->wkv_all)
  const float *bq_c = nullptr, *bo_c = nullptr, *g3 = nullptr, *be3 = nullptr;
  CUtensorMap m_wq_c, m_wo_c_256;
  // trans_dec with a CLIP memory: the value rows W_v [d, d], b_v and W_o of multihead_attn in fp32 (weight store)
  const float *wv_c32 = nullptr, *bv_c32 = nullptr, *wo_c32 = nullptr;
};

struct GraphKey {
  int mode = -1, B = 0, T = 0, flags = 0;
  int order = 0;                    // PLMS (Adams-Bashforth step): the order; 0 for DDPM / DDIM
  const void *pred = nullptr, *imask = nullptr, *iweight = nullptr, *imotion = nullptr;
  const void* target_g = nullptr;   // the workspace's target embedding, or nullptr when the loop has no target
  const void* hs = nullptr;         // the workspace's handshake descriptor, or nullptr when the loop has none
  int guide = -1;                   // joint-position control: the step ends in GUIDE_VARIANTS[guide] (-1: unguided)
  int chars = 0;                    //     in clusters of `chars` CTAs
  int groups = 0;                   // multi-prompt guidance: the step ends in compose_step_kernel over G groups
  bool slots = false;               // continuous batching: a schedule index per row (b200mdm_slots_begin)
  bool operator==(const GraphKey& o) const {
    return mode == o.mode && B == o.B && T == o.T && flags == o.flags && order == o.order && pred == o.pred &&
           imask == o.imask && iweight == o.iweight && imotion == o.imotion && target_g == o.target_g && hs == o.hs &&
           guide == o.guide && chars == o.chars && groups == o.groups && slots == o.slots;
  }
};

// Everything sized by (batch, nframes, CFG halves): activations, their TMA maps, the conditioning rows and the captured
// step graph (whose kernel parameters are these very pointers).  The engine keeps the workspace in use as its own
// base-class fields and parks the others in a small pool, so callers that alternate between shapes (the evaluation
// loader: 32 <-> 32 x mm_num_repeats, comp_v6_model_dataset.py:148-256) neither re-allocate nor re-capture.
struct Workspace {
  int B = 0, T = 0, S = 0, halves = 1, Bp = 0, M = 0, MB = 0;
  // multi-prompt guidance (b200mdm_set_cond_multi*): G = K + 1 groups of B motions, Bp = G * B, the unconditional group
  // last; 0 for the plain / CFG batch of `halves`.  g16 then holds the frame rows of every group, and mp_x0
  // [G, B, JF, T] the raw x0 of every group, which compose_step_kernel composes.
  int groups = 0;
  float* mp_x0 = nullptr;
  __half *xin16 = nullptr, *hres = nullptr, *qkv16 = nullptr, *att16 = nullptr, *ffn16 = nullptr, *g16 = nullptr;
  float *tok0 = nullptr, *condproj = nullptr, *proj = nullptr, *scale = nullptr, *x_work = nullptr, *eps_buf = nullptr;
  int *kvlen = nullptr, *tvec = nullptr, *action = nullptr;
  CUtensorMap m_xin, m_h16, m_att, m_ffn, m_g16;      // A operands (loads, box 128 rows)
  CUtensorMap m_qkv_st, m_ffn_st;                      // epilogue slabs (box 32 rows x 128 bytes)
  CUtensorMap m_qkv_kv;                                // attention core: per-sample K / V tiles of qkv16 (box all keys)
  CUtensorMap m_res_c, m_res_u;                        // per-CFG-half views of the residual stream (embedding epilogue)
  CUtensorMap m_hres;                                  // the whole residual stream [M, 2d], box 64 x 64 (residual + LayerNorm)
  float* pe_bias = nullptr;
  bool cond_set = false;
  // trans_dec (DiP): prefix frames + text-token memory
  int Mt = 0;
  float *encperm = nullptr, *memtok = nullptr, *memproj = nullptr;   // [B*Mt, cond_dim], [B*Mt, d], [Bp*Mt, d]
  __half *mem16 = nullptr, *qc16 = nullptr, *kvc16 = nullptr;        // [Bp*Mt, d], [M, d], [Bp*Mt, 2d]
  unsigned char* memmask = nullptr;                                   // [Bp, Mt] 1 = padding
  CUtensorMap m_mem, m_qc_st, m_kvc_st;
  bool prefix_set = false;
  // trans_dec with a CLIP memory (kernels.cuh, cross_rows_kernel): the memory rows' per-sample part mb [Bp, d], a GEMV
  // scratch [Bp, d], cb [L, Bp, d] (per loop) and the step's cross-attention rows c [L, Bp, d]
  float *cross_mb = nullptr, *cross_u = nullptr, *cross_b = nullptr, *cross_c = nullptr;
  // target-location conditioning: validity [B, n_ext] (1.0 / 0.0) and g = embed_target_cond(...) [B, d], read by both
  // CFG halves; target_set is cleared by every b200mdm_set_cond* call
  float *tgt_valid = nullptr, *tgt_g = nullptr;
  bool target_set = false;
  // handshakes between chained windows (b200mdm_set_handshake): the blend kernel's descriptor [1 + 2B] int32 (layout
  // HS_* in kernels.cuh), allocated on first use; hs_set is cleared by every b200mdm_set_cond* call
  int* hs_desc = nullptr;
  bool hs_set = false;
  // joint-position control (b200mdm_set_joint_guidance): the raw x0 [B, JF, T] the output GEMM hands to the guidance
  // kernel, allocated on first use
  float* jg_x0 = nullptr;
  // PLMS, allocated on first use: eps history ring [PLMS_RING, B, JF, T], the improved-Euler step's mean1 (the input of
  // its second forward) and its first x0.  plms_done = evaluations of the PLMS loop in flight (-1: none to continue).
  float *plms_ring = nullptr, *plms_mid = nullptr, *plms_pred = nullptr;
  int plms_done = -1, plms_order = 0;
  // DPM-Solver++, allocated on first use: x0 history [DPM_SLOTS, B, JF, T].  dpm_done = evaluations of the DPM loop in
  // flight (-1: none to continue).
  float* dpm_hist = nullptr;
  int dpm_done = -1, dpm_order = 0;
  // variational-bound loop, allocated on first use: x_start [B, JF, T] (the loop state, never overwritten), the
  // per-(row, 32-column chunk) sums of the output epilogue [VB_TERMS, B*T, vb_chunks] and the per-step means
  // [VB_TERMS, B, vb_cap] (column n_steps - 1 - i for schedule index i).  vb_live: a bound loop that may be continued.
  float *vb_xs = nullptr, *vb_part = nullptr, *vb_terms = nullptr;
  int vb_cap = 0;
  bool vb_live = false;
  // continuous batching (b200mdm_slots_begin), allocated on first use: the per-row slot state [B], read and written
  // inside the step graph (epilogues.cuh, SlotState)
  SlotState* slots = nullptr;
  // captured step graph of this workspace
  cudaGraphExec_t graph_exec = nullptr;
  GraphKey graph_key;
  int graph_kernels = 0;
  unsigned long long last_use = 0;
};

struct b200mdm_engine : Workspace {
  b200mdm_config cfg;
  int d, ff, L, H, JF, Kp_in, N_out_pad;
  int num_sms = 132;
  std::map<std::string, Tensor32> store;
  bool finalized = false;
  // repacked weights
  __half *w_in3 = nullptr, *w_out3 = nullptr;
  CUtensorMap m_win, m_wout;
  std::vector<LayerW> layers;
  const float *b_in = nullptr, *b_out = nullptr, *pe = nullptr, *w_txt = nullptr, *b_txt = nullptr, *act_emb = nullptr;
  float *temb_hidden = nullptr, *temb_table = nullptr;
  // trans_dec: key/value projection rows of the cross-attention of ALL layers, [L * 2d, d] fp16 + bias [L * 2d]: the text
  // memory is the same for every layer, so one GEMM per step projects it for all of them
  __half* wkv_all = nullptr;
  float* bkv_all = nullptr;
  CUtensorMap m_wkv_all;
  // target encoder, packed for target_embed_kernel (kernels.cuh): G groups of width tdj, first layer tin wide
  float *tw0 = nullptr, *tb0 = nullptr, *twk = nullptr, *tbk = nullptr, *twsum = nullptr;
  int tG = 0, tdj = 0, tin = 0, tlayers = 0;
  std::vector<float> h_valid;
  // schedule: the row tables (SchedTable) and the timestep map, allocated once at `sched_cap` rows (the step graphs
  // hold these pointers).  Every b200mdm_set_schedule makes the tables after TAB_STEP stale until their own setter.
  float* tab[N_TABLES] = {};
  bool tab_fresh[N_TABLES] = {};
  int* tmap = nullptr;
  int n_steps = 0, sched_cap = 0;
  // parked workspaces (see Workspace)
  std::vector<Workspace> pool;
  unsigned long long use_clock = 0;
  // host staging for b200mdm_set_cond* (kept alive until the next call: no stream synchronisation needed)
  std::vector<int> h_kv, h_action;
  std::vector<unsigned char> h_mask;
  std::vector<int> h_hs;
  // trans_dec (DiP)
  bool dec = false;
  // trans_dec with emb_trans_dec and a CLIP memory: sequence = timestep token + frames, cross-attention = a per-sample
  // row (kernels.cuh, cross_rows_kernel); cross_t = W_o,l W_v,l temb[t] for every layer and model timestep [L, R, d]
  bool dec_clip = false;
  float* cross_t = nullptr;
  int ctx = 0, s_off = 1;
  int kw = 1;   // 2: fp16 activations between the layer GEMMs are [hi | lo] pairs along K (trans_dec engine)
  const unsigned char* inpaint_mask = nullptr;
  const float* inpaint_weight = nullptr;   // soft inpainting (b200mdm_set_inpaint_weight); never set with the mask
  const float* inpaint_motion = nullptr;
  // joint-position control and the terms that extend it (b200mdm_set_{joint,foot,scene,interaction}_guidance): the
  // device descriptor (read by the step graph at every replay, allocated on first use), its host staging h_guide, which
  // every setter uploads whole, and the terms on (GuideTerm bits), which every b200mdm_set_cond* call clears and each
  // setter clears from its own term up.  h_guide.f keeps the lengths of a foot call with both weights 0 and h_guide.s
  // the grids of a scene call that turned its terms off: the terms above them read both.  The lengths and the reach rows
  // the descriptor points to live in fg_len [fg_len_cap] int32 and ig_pairs [ig_pairs_cap] (device, allocated on first
  // use), staged from h_fg_len and h_ig_pairs.
  GuideDesc* jg_desc = nullptr;
  GuideDesc h_guide{};
  unsigned guide_terms = 0;
  int* fg_len = nullptr;
  int fg_len_cap = 0;
  std::vector<int> h_fg_len;
  InterPair* ig_pairs = nullptr;
  int ig_pairs_cap = 0;
  std::vector<InterPair> h_ig_pairs;
  // multi-prompt guidance: the prompt-weight descriptor (read by the step graph at every replay, allocated on first
  // use) and its host staging; pw_set is cleared by every b200mdm_set_cond* call
  PromptWeight* pw_desc = nullptr;
  PromptWeight h_pw{};
  bool pw_set = false;
  // in-engine noise (B200MDM_FLAG_PHILOX_NOISE): counter-based Philox4x32-10 keyed by (seed, schedule index, global sample)
  unsigned long long noise_seed = 0;
  long long noise_sample_base = 0;
  // loop machinery
  StepState* state = nullptr;   // device-side step counter + per-loop noise description, shared by every workspace
  cudaStream_t work = nullptr;
  cudaEvent_t ev_in = nullptr, ev_out = nullptr;
  long long launches = 0;
  // DiP: whether b200mdm_set_cond_dec filled the memory's conditional rows with the unconditional projection
  bool mem_uncond = false;
  // autoregressive chain (b200mdm_chain_setup): per-chunk projected memories [n, Bp*Mt, d] and masks [n, Bp*Mt] (unused
  // when every chunk keeps the memory of b200mdm_set_cond_dec), the prefix handed on [B, JF, ctx], the layout, and the
  // global step the next b200mdm_chain_loop_range must start at (-1: no chain to run or continue)
  float *chain_mem = nullptr, *chain_prefix = nullptr;
  unsigned char* chain_mask = nullptr;
  size_t chain_mem_cap = 0, chain_mask_cap = 0, chain_prefix_cap = 0;
  std::vector<unsigned char> h_chain_mask;
  int chain_n = 0, chain_off = 0, chain_crop = 0, chain_next = -1;
  bool chain_mems = false;
  // the prefix of b200mdm_set_prefix (caller-owned), which b200mdm_chain_set_goal reads under include_prefix
  const float* prefix_src = nullptr;
  // continuous batching on the workspace in use (b200mdm_slots_begin .. the next b200mdm_set_cond*): the sampler and
  // flags of the session, and per slot whether it holds a request not yet read and how many of its steps are still to
  // run -- the host knows when each slot finishes without asking the device
  bool slot_mode = false;
  int slot_sampler = 0, slot_flags = 0;
  std::vector<unsigned char> slot_busy;
  std::vector<int> slot_left;
  std::vector<int> h_slot_idx;   // host staging of b200mdm_sample_step_at's indices
  // a token-memory session (b200mdm_chain_slots_begin; slot_mode on a BERT-memory engine): per slot, what its hand-offs
  // need -- its Philox key, scale and valid keys to re-arm it, its motion length, first output frame and chunk position
  struct ChainSlot {
    unsigned long long seed = 0;
    long long g = 0;
    float scale = 0.f;
    int kv = 0, length = 0, off = 0, chunk = 0, n_chunks = 0;
  };
  std::vector<ChainSlot> chain_slot;
  // a goal-directed chain (b200mdm_chain_set_goal): the caller's mean / std [JF] and goals [n_goals, B, n_ext, 3], the
  // per-sample carry [B, CF_CARRY] and the next chunk's target [B, n_ext, 3]; live while goal_set and the chain is
  // (chain_setup clears goal_set, and everything that ends a chain sets chain_next = -1)
  const float *goal_mean = nullptr, *goal_std = nullptr, *goal_src = nullptr;
  double* goal_carry = nullptr;
  float* goal_tgt = nullptr;
  size_t goal_carry_cap = 0, goal_tgt_cap = 0;
  int goal_n = 0;
  bool goal_set = false;
};

template <class T>
static int dalloc(T** p, size_t n, bool zero = false) {
  const cudaError_t err = cudaMalloc(reinterpret_cast<void**>(p), n * sizeof(T));
  if (err != cudaSuccess) {
    cudaGetLastError();   // an out-of-memory error is not sticky: clear it so that later launches do not report it
    return fail(B200MDM_ECUDA, "cudaMalloc of %zu bytes failed: %s", n * sizeof(T), cudaGetErrorString(err));
  }
  if (zero) CUDA_TRY(cudaMemset(*p, 0, n * sizeof(T)));
  return B200MDM_OK;
}
template <class T>
static void dfree(T*& p) {
  if (p) cudaFree(p);
  p = nullptr;
}

// ------------------------------------------------------------------------------------------------ launchers
template <int BN, class Epi>
static int set_gemm_attr() {
  CUDA_TRY(cudaFuncSetAttribute(gemm_f16_wgmma<BN, Epi>, cudaFuncAttributeMaxDynamicSharedMemorySize, GemmSmem<BN, Epi>::TOTAL));
  return B200MDM_OK;
}
template <class Epi>
static int set_pingpong_attr() {
  CUDA_TRY(cudaFuncSetAttribute(gemm_f16_pingpong<Epi>, cudaFuncAttributeMaxDynamicSharedMemorySize, PP_SMEM_BYTES));
  return B200MDM_OK;
}
template <int KEYS>
static int set_attention_attr() {
  CUDA_TRY(cudaFuncSetAttribute(attention_tc_kernel<KEYS, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                AttnTcSmem::total(KEYS)));
  CUDA_TRY(cudaFuncSetAttribute(attention_tc_kernel<KEYS, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                AttnTcSmem::total(KEYS)));
  return B200MDM_OK;
}

// The terms of joint-position control, as bits of b200mdm_engine::guide_terms; each extends the ones below it
enum GuideTerm : unsigned { GT_JOINT = 1, GT_FOOT = 2, GT_SCENE = 4, GT_INTER = 8 };
// The guidance kernels, one row per highest term on (guide_variant): the step kernel, the test kernel of the
// b200mdm_test_*_guidance hooks, their dynamic shared memory (T, R) and whether they run in clusters of the
// descriptor's `chars` CTAs
struct GuideVariant {
  void (*step)(const GuideDesc*, const float*, EpiOutParams);
  void (*test)(GuideDesc, const float*, float*, float*, int, int, int);
  size_t (*smem)(int, int);
  bool clusters;
};
static const GuideVariant GUIDE_VARIANTS[] = {
    {joint_guidance_step_kernel<false, false>, joint_guidance_test_kernel<false, false>, jg_smem_bytes, false},
    {joint_guidance_step_kernel<true, false>, joint_guidance_test_kernel<true, false>, fg_smem_bytes, false},
    {joint_guidance_step_kernel<true, true>, joint_guidance_test_kernel<true, true>, fg_smem_bytes, false},
    {joint_guidance_step_kernel<true, true, true>, joint_guidance_test_kernel<true, true, true>, ig_smem_bytes, true},
};
// the row of GUIDE_VARIANTS of the terms on (-1: none)
static int guide_variant(unsigned terms) { return terms ? 31 - __builtin_clz(terms) : -1; }
// The joints J and ric features R = 4 + 3 (J - 1) of a model the guidance accepts: HumanML3D (D = 263) or KIT (D = 251)
struct RicDims {
  int J, R;
};
static RicDims ric_dims(int D) {
  const int J = D == 263 ? 22 : 21;
  return {J, 4 + 3 * (J - 1)};
}

static int init_kernel_attrs() {
  // function attributes are per device: track which ordinals have been initialised
  static unsigned long long done_mask = 0;
  int dev = 0;
  CUDA_TRY(cudaGetDevice(&dev));
  if (dev < 64 && ((done_mask >> dev) & 1ull)) return B200MDM_OK;
  TRY((set_pingpong_attr<EpiBiasF16<false>>()));
  TRY((set_pingpong_attr<EpiBiasF16<true>>()));
  TRY((set_pingpong_attr<EpiBiasF16Wide<true>>()));
  TRY((set_pingpong_attr<EpiBiasF16Global>()));
  CUDA_TRY(cudaFuncSetAttribute(gemm_resid_ln_cluster, cudaFuncAttributeMaxDynamicSharedMemorySize, GemmLnSmem::TOTAL));
  TRY((set_gemm_attr<128, EpiEmbed>()));
  TRY((set_gemm_attr<96, EpiOut<OutStep>>()));
  TRY((set_gemm_attr<96, EpiOut<OutStepSlots>>()));
  TRY((set_gemm_attr<96, EpiOut<OutPlms>>()));
  TRY((set_gemm_attr<96, EpiOut<OutReverse>>()));
  TRY((set_gemm_attr<96, EpiOut<OutDpm>>()));
  TRY((set_gemm_attr<96, EpiOut<OutVb>>()));
  TRY((set_attention_attr<64>()));
  TRY((set_attention_attr<208>()));
  TRY((set_attention_attr<256>()));
  CUDA_TRY(cudaFuncSetAttribute(cross_attention_long_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, XAL_SMEM));
  for (const GuideVariant& v : GUIDE_VARIANTS) {
    const int smem = static_cast<int>(v.smem(JG_MAX_FRAMES, JG_MAX_FEATS));
    CUDA_TRY(cudaFuncSetAttribute(v.step, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    CUDA_TRY(cudaFuncSetAttribute(v.test, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  }
  if (dev < 64) done_mask |= 1ull << dev;
  return B200MDM_OK;
}

// ------------------------------------------------------------------------------------------------ launches
// Kernels of the sampling step are launched with programmatic stream serialization (PDL): the next kernel's CTAs are
// scheduled as SMs drain and run their prologue (barrier init, descriptor prefetch, bias staging)
// under the tail of the current one; every kernel calls griddepcontrol.wait before it touches global data.
// B200MDM_PDL=0 in the environment restores plain stream order.
static bool g_pdl_now = false;   // set while b200mdm is enqueueing a step
static bool pdl_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("B200MDM_PDL");
    v = (e && e[0] == '0') ? 0 : 1;
  }
  return v == 1;
}
struct PdlScope {
  PdlScope() { g_pdl_now = pdl_enabled(); }
  ~PdlScope() { g_pdl_now = false; }
};
// cluster > 0: thread-block clusters of `cluster` CTAs along x
template <class... KArgs, class... Args>
static cudaError_t launch_kc(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, int cluster,
                             Args&&... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute at[2];
  int n = 0;
  if (cluster > 0) {
    at[n].id = cudaLaunchAttributeClusterDimension;
    at[n].val.clusterDim.x = static_cast<unsigned>(cluster);
    at[n].val.clusterDim.y = 1;
    at[n].val.clusterDim.z = 1;
    ++n;
  }
  if (g_pdl_now) {
    at[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  cfg.attrs = at;
  cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(std::forward<Args>(args))...);
}
template <class... KArgs, class... Args>
static cudaError_t launch_k(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args&&... args) {
  return launch_kc(kern, grid, block, smem, s, 0, std::forward<Args>(args)...);
}

template <class Epi, class = void> struct epi_unstaged : std::false_type {};
template <class Epi> struct epi_unstaged<Epi, std::enable_if_t<Epi::UNSTAGED>> : std::true_type {};

// the staged GEMM (gemm.cuh) of the embedding and the output projection; the speed of both was measured with these
// pipeline depths
static_assert(GemmSmem<128, EpiEmbed>::STAGES == 2, "shared-memory budget: 2 operand stages for the embedding GEMM");
static_assert(GemmSmem<96, EpiOut<OutStep>>::STAGES == 5, "shared-memory budget: 5 operand stages for the output GEMM");
template <int BN, class Epi>
static int launch_gemm(const CUtensorMap& a, const CUtensorMap& b, int M, int N, int K, const typename Epi::Params& p,
                       cudaStream_t s, int num_sms) {
  const int tiles = ((M + GEMM_BLOCK_M - 1) / GEMM_BLOCK_M) * ((N + BN - 1) / BN);
  const int grid = tiles < num_sms ? tiles : num_sms;
  CUDA_TRY(launch_k(gemm_f16_wgmma<BN, Epi>, dim3(grid), dim3(GEMM_THREADS), GemmSmem<BN, Epi>::TOTAL, s, a, b, M, N, K, p));
  return B200MDM_OK;
}
// projection GEMMs of the step (gemm_pingpong.cuh): 128 x 128 tiles, the two consumer warpgroups take turns (b: W map
// with box 128 rows; c: output map with box 32 rows x 64 columns)
template <class Epi>
static int launch_gemm_pp(const CUtensorMap& a, const CUtensorMap& b, const CUtensorMap& c, int M, int N, int K,
                          const typename Epi::Params& p, cudaStream_t s, int num_sms) {
  if (!epi_unstaged<Epi>::value && N * 4 > GEMM_BIAS_BYTES)
    return fail(B200MDM_ENOTIMPL, "GEMM epilogue vectors are staged for N <= %d", GEMM_BIAS_BYTES / 4);
  const int tiles = ((M + GEMM_BLOCK_M - 1) / GEMM_BLOCK_M) * ((N + PP_BLOCK_N - 1) / PP_BLOCK_N);
  const int grid = tiles < num_sms ? tiles : num_sms;
  CUDA_TRY(launch_k(gemm_f16_pingpong<Epi>, dim3(grid), dim3(GEMM_THREADS), PP_SMEM_BYTES, s, a, b, c, M, N, K, p));
  return B200MDM_OK;
}
// out16 = fp16(act(A W^T + bias))
template <bool GELU>
static int launch_gemm_bias(const CUtensorMap& a, const CUtensorMap& b, const CUtensorMap& c, int M, int N, int K,
                            const float* bias, cudaStream_t s, int num_sms) {
  typename EpiBiasF16<GELU>::Params p{bias};
  return launch_gemm_pp<EpiBiasF16<GELU>>(a, b, c, M, N, K, p, s, num_sms);
}

// h <- LayerNorm(h + A W^T + bias), 2-CTA cluster splitting the 512 columns, LayerNorm statistics exchanged through
// distributed shared memory (w256: W map with box 256 rows; hres: map of the residual stream [M, 2 x 512] fp16 with
// box GLN_RES_BOX_ROWS rows x 64 columns, make_hres_map)
static int launch_gemm_resid_ln(const CUtensorMap& a, const CUtensorMap& w256, const CUtensorMap& hres, int M, int K,
                                const float* bias, const float* gamma, const float* beta, cudaStream_t s, int num_sms) {
  const int tiles = (M + GEMM_BLOCK_M - 1) / GEMM_BLOCK_M;
  const int max_clusters = num_sms / 2;
  const int clusters = tiles < max_clusters ? tiles : max_clusters;
  GemmLnParams lp{bias, gamma, beta, 1e-5f};
  CUDA_TRY(launch_k(gemm_resid_ln_cluster, dim3(2 * clusters), dim3(GLN_THREADS), GemmLnSmem::TOTAL, s, a, w256, hres, M, K, lp));
  return B200MDM_OK;
}

// attention core for sequences of up to 256 tokens (every configuration of the reference: 197 / 61 / 60)
// map_kv: qkv viewed per sample, box {64, atc_keys(S), 1} (make_attention_kv_map)
static int make_attention_kv_map(CUtensorMap* m, const void* qkv, int n_samples, int S, int ld) {
  return make_map_3d(m, qkv, n_samples, S, ld, ld, atc_keys(S));
}
template <int KEYS>
static cudaError_t launch_attention_keys(const CUtensorMap& map_kv, const __half* qkv, __half* out, const int* kvlen,
                                         dim3 grid, int S, int d, float scale_log2, cudaStream_t s, bool wide) {
  return launch_k(wide ? attention_tc_kernel<KEYS, true> : attention_tc_kernel<KEYS, false>, grid, dim3(ATC_THREADS),
                  AttnTcSmem::total(KEYS), s, map_kv, qkv, out, kvlen, S, d, scale_log2);
}
static int launch_attention_tc(const CUtensorMap& map_kv, const __half* qkv, __half* out, const int* kvlen, int n_samples,
                               int S, int d, int H, cudaStream_t s, bool wide = false) {
  if (d != H * ATC_DH) return fail(B200MDM_ENOTIMPL, "attention: head_dim must be 128");
  if (S > ATC_MAX_KEYS) return fail(B200MDM_ENOTIMPL, "attention: at most %d tokens per sample", ATC_MAX_KEYS);
  const float scale_log2 = 1.4426950408889634f / sqrtf(static_cast<float>(ATC_DH));
  const int tiles = (S + ATC_QROWS - 1) / ATC_QROWS;
  const dim3 grid(H, n_samples, (tiles + ATC_TILES_PER_CTA - 1) / ATC_TILES_PER_CTA);
  const int keys = atc_keys(S);
  if (keys == 64) CUDA_TRY(launch_attention_keys<64>(map_kv, qkv, out, kvlen, grid, S, d, scale_log2, s, wide));
  else if (keys == 208) CUDA_TRY(launch_attention_keys<208>(map_kv, qkv, out, kvlen, grid, S, d, scale_log2, s, wide));
  else CUDA_TRY(launch_attention_keys<256>(map_kv, qkv, out, kvlen, grid, S, d, scale_log2, s, wide));
  return B200MDM_OK;
}
// cross-attention core of a trans_dec layer over a text memory of Mt tokens: q16 [n*S, d]; kv rows (sample, token) of
// pitch ld_kv holding k | v; mask [n, Mt], 1 = padding.  Up to 64 tokens every key of a head sits in registers, longer
// memories take the key-blocked kernel.
static int launch_cross_attention(const __half* q16, const __half* kv, const unsigned char* mask, __half* out, int n_samples,
                                  int S, int Mt, int d, int H, int ld_kv, cudaStream_t s) {
  const float sl2 = 1.4426950408889634f / sqrtf(128.0f);
  const dim3 cg(H, n_samples), cb(128);
  if (Mt <= 16)
    CUDA_TRY(launch_k(cross_attention_kernel<2>, cg, cb, 0, s, q16, kv, mask, out, S, Mt, d, ld_kv, sl2));
  else if (Mt <= 32)
    CUDA_TRY(launch_k(cross_attention_kernel<4>, cg, cb, 0, s, q16, kv, mask, out, S, Mt, d, ld_kv, sl2));
  else if (Mt <= 64)
    CUDA_TRY(launch_k(cross_attention_kernel<8>, cg, cb, 0, s, q16, kv, mask, out, S, Mt, d, ld_kv, sl2));
  else
    CUDA_TRY(launch_k(cross_attention_long_kernel, dim3(H, n_samples, (S + XAL_ROWS - 1) / XAL_ROWS), cb, XAL_SMEM, s, q16, kv,
                      mask, out, S, Mt, d, ld_kv, sl2));
  return B200MDM_OK;
}
// h <- LayerNorm(h + c[row / S]) over the [hi | lo] residual stream (the CLIP decoder's one-token cross-attention block)
static int launch_row_bias_ln(__half* hres, const float* c, const float* gamma, const float* beta, int M, int S, cudaStream_t s) {
  CUDA_TRY(launch_k(row_bias_ln_kernel, dim3((M + RBLN_ROWS_PER_CTA - 1) / RBLN_ROWS_PER_CTA), dim3(32 * RBLN_ROWS_PER_CTA), 0, s,
                    hres, c, gamma, beta, M, S, 1e-5f));
  return B200MDM_OK;
}
// grid of the Philox kernels over B samples of n elements (256 threads, one quad each, grid-stride beyond 1184 blocks)
static int philox_blocks(int B, long long n) {
  const long long quads = (n + 3) / 4 * B;
  return static_cast<int>(quads / 256 + 1 < 1184 ? quads / 256 + 1 : 1184);
}
// eps [B, n] of the counter-based noise stream; state != nullptr: seed, sample base and step come from the step state
static int launch_philox(float* out, int B, long long n, unsigned long long seed, long long sample_base, uint32_t step_id,
                         const StepState* state, cudaStream_t s) {
  CUDA_TRY(launch_k(philox_normal_kernel, dim3(philox_blocks(B, n)), dim3(256), 0, s, out, B, n, seed, sample_base, step_id,
                    state));
  return B200MDM_OK;
}
// x [B, JF, cols] -> rows row_off .. row_off + cols of every S-row sequence of the embedding GEMM's A operand [hi | lo | hi]
static int launch_pack_input(const float* x, __half* xin16, int B, int JF, int cols, int S, int Kp, int row_off, cudaStream_t s) {
  CUDA_TRY(launch_k(pack_input_kernel, dim3((cols + 31) / 32, (JF + 31) / 32, B), dim3(32, 8), 0, s, x, xin16, B, JF, cols, S,
                    Kp, 3 * Kp, row_off));
  return B200MDM_OK;
}
// residual stream <- xin16 W_in3^T + pe_bias[s], stored to the rows of both CFG halves (EpiEmbed)
static int launch_embed_gemm(const CUtensorMap& m_xin, const CUtensorMap& m_win, const CUtensorMap& m_res_c,
                             const CUtensorMap& m_res_u, const float* pe_bias, int MB, int S, int d, int Kp, int halves,
                             cudaStream_t s, int num_sms) {
  EpiEmbed::Params p;
  p.res_c = m_res_c; p.res_u = m_res_u;
  p.pe_bias = pe_bias;
  p.S = S; p.d = d; p.halves = halves;
  return launch_gemm<128, EpiEmbed>(m_xin, m_win, MB, d, 3 * Kp, p, s, num_sms);
}
// the bound step's x_t into x_t [B, n] from x_start and the step's eps (noise, or the tape of the step state)
static int launch_vb_xt(float* x_t, const float* x_start, const float* noise, const float* sched_vb, const StepState* state,
                        size_t n, cudaStream_t s) {
  const int blocks = static_cast<int>(n / 256 + 1 < 1184 ? n / 256 + 1 : 1184);
  CUDA_TRY(launch_k(vb_xt_kernel, dim3(blocks), dim3(256), 0, s, x_t, x_start, noise, sched_vb, state, n));
  return B200MDM_OK;
}
// the bound step's per-sample means of its three terms from the epilogue's partial sums -> column n_steps - 1 - cur of terms
static int launch_vb_reduce(float* terms, int ld_terms, const float* part, int B, int T, int JF, const StepState* state,
                            cudaStream_t s) {
  CUDA_TRY(launch_k(vb_reduce_kernel, dim3(B, VB_TERMS), dim3(VB_REDUCE_THREADS), 0, s, terms, ld_terms, part, B,
                    T * ((JF + 31) / 32), static_cast<float>(JF) * static_cast<float>(T), state));
  return B200MDM_OK;
}
// g16 [B*T, 3d] = [hi | hi | lo] of the CFG blend of the frame rows of hres, with the handshakes of descriptor hs
// (nullptr: none)
static int launch_blend_split(const __half* hres, __half* g16, const float* scale, int B, int S, int T, int s_off, int d,
                              int halves, const int* hs, cudaStream_t s) {
  CUDA_TRY(launch_k(blend_split_kernel, dim3((B * T + 7) / 8), dim3(256), 0, s, hres, g16, scale, B, S, T, s_off, d, halves, hs));
  return B200MDM_OK;
}

// The blend kernel's handshake descriptor (HS_* in kernels.cuh) for B windows of T frames: window b has lengths[b]
// frames (all T without lengths) and continues window b - 1 unless motion_start[b] (without motion_start, the batch is
// one motion).  desc is left empty when nothing is blended (h == 0, or every window begins a motion).  Host-only: bad
// arguments return B200MDM_EINVAL before any CUDA call.
static int handshake_desc(int h, int B, int T, const int64_t* lengths, const uint8_t* motion_start, std::vector<int>* desc) {
  desc->clear();
  if (h < 0) return fail(B200MDM_EINVAL, "handshake size %d < 0", h);
  if (B <= 0 || T <= 0) return fail(B200MDM_EINVAL, "bad batch / nframes");
  if (motion_start && !motion_start[0]) return fail(B200MDM_EINVAL, "window 0 must begin a motion (motion_start[0])");
  if (h == 0) return B200MDM_OK;
  std::vector<int> d(1 + 2 * static_cast<size_t>(B), 0);
  d[HS_H] = h;
  bool any = false;
  for (int b = 0; b < B; ++b) {
    const long long n = lengths ? lengths[b] : T;
    if (n < 0 || n > T) return fail(B200MDM_EINVAL, "window %d: length %lld outside [0, %d]", b, n, T);
    d[HS_LEN(b)] = static_cast<int>(n);
    d[HS_CHAIN(b)] = (b > 0 && !(motion_start && motion_start[b])) ? 1 : 0;
    any = any || d[HS_CHAIN(b)];
  }
  for (int b = 0; b < B; ++b) {
    const bool prev = d[HS_CHAIN(b)] != 0, next = b + 1 < B && d[HS_CHAIN(b + 1)] != 0;
    const int n = d[HS_LEN(b)];
    if ((prev || next) && n < h) return fail(B200MDM_EINVAL, "chained window %d has %d frames < handshake size %d", b, n, h);
    if (prev && next && n < 2 * h)
      return fail(B200MDM_EINVAL, "window %d has %d frames < 2 x handshake size %d: its two handshakes would overlap", b, n, h);
  }
  if (any) desc->swap(d);
  return B200MDM_OK;
}
#ifdef B200_TRACE
// Instrumented build only (lib/libb200mdm_trace.so): B200MDM_DEBUG_SKIP is a bit mask of layer kernels to leave out of the
// step (1 attention, 2 out-proj+LN, 4 FFN-up, 8 FFN-down+LN) -- the results are garbage, the loop time difference is what
// that kernel costs INSIDE the graph loop (programmatic dependent launch, L2 window), which no profiler shows.
static int debug_skip_mask() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("B200MDM_DEBUG_SKIP");
    v = e ? atoi(e) : 0;
  }
  return v;
}
#define B200_SKIP(bit) (debug_skip_mask() & (bit))
#else
#define B200_SKIP(bit) (0)
#endif
// ------------------------------------------------------------------------------------------------ API: basics
extern "C" const char* b200mdm_last_error(void) { return g_err; }
extern "C" int b200mdm_version(void) { return 1; }

extern "C" int b200mdm_create(const b200mdm_config* cfg, b200mdm_engine** out) {
  if (!cfg || !out) return fail(B200MDM_EINVAL, "null argument");
  if (cfg->arch != B200MDM_ARCH_TRANS_ENC && cfg->arch != B200MDM_ARCH_TRANS_DEC)
    return fail(B200MDM_ENOTIMPL, "arch %d: trans_enc and trans_dec are implemented", cfg->arch);
  if (cfg->arch == B200MDM_ARCH_TRANS_DEC && (cfg->cond_mode != B200MDM_COND_TEXT || cfg->context_len < 0))
    return fail(B200MDM_ENOTIMPL, "trans_dec needs text-token conditioning (BERT) and context_len >= 0");
  if (cfg->emb_trans_dec < 0 || cfg->emb_trans_dec > 1 || cfg->dec_memory < B200MDM_DEC_MEMORY_TOKENS ||
      cfg->dec_memory > B200MDM_DEC_MEMORY_CLIP)
    return fail(B200MDM_EINVAL, "emb_trans_dec must be 0 or 1 and dec_memory 0 (tokens) or 1 (CLIP) (got %d / %d)",
                cfg->emb_trans_dec, cfg->dec_memory);
  if (cfg->arch == B200MDM_ARCH_TRANS_ENC && (cfg->emb_trans_dec || cfg->dec_memory))
    return fail(B200MDM_EINVAL, "emb_trans_dec and dec_memory are trans_dec fields");
  if (cfg->arch == B200MDM_ARCH_TRANS_DEC && (cfg->dec_memory == B200MDM_DEC_MEMORY_CLIP) != (cfg->emb_trans_dec == 1))
    return fail(B200MDM_ENOTIMPL, "trans_dec implements the BERT token memory without the timestep token (DiP) and the CLIP "
                "memory with it (emb_trans_dec); got dec_memory %d, emb_trans_dec %d", cfg->dec_memory, cfg->emb_trans_dec);
  if (cfg->dec_memory == B200MDM_DEC_MEMORY_CLIP && cfg->context_len != 0)
    return fail(B200MDM_ENOTIMPL, "trans_dec with a CLIP memory has no prefix completion (context_len %d)", cfg->context_len);
  if (cfg->latent_dim != 512 || cfg->num_heads != 4 || cfg->ff_size % 64 || cfg->ff_size <= 0)
    return fail(B200MDM_ENOTIMPL, "kernels are specialised for latent_dim 512 / 4 heads (got %d / %d)", cfg->latent_dim,
                cfg->num_heads);
  if (cfg->num_layers <= 0 || cfg->njoints <= 0 || cfg->nfeats <= 0 || cfg->pos_embed_max_len <= 0 || cfg->temb_rows <= 0)
    return fail(B200MDM_EINVAL, "bad config");
  if (cfg->target_encoder < B200MDM_TARGET_NONE || cfg->target_encoder > B200MDM_TARGET_SPLIT)
    return fail(B200MDM_EINVAL, "target_encoder %d: 0 none, 1 single, 2 multi, 3 split", cfg->target_encoder);
  if (cfg->target_encoder != B200MDM_TARGET_NONE) {
    if (cfg->target_joints <= 0 || cfg->target_joints > 64 || cfg->target_enc_layers < 0 || cfg->target_enc_layers > 16)
      return fail(B200MDM_EINVAL, "target encoder: 1..64 joints and 0..16 layers (got %d / %d)", cfg->target_joints,
                  cfg->target_enc_layers);
    if (cfg->target_encoder == B200MDM_TARGET_SPLIT && cfg->latent_dim % cfg->target_joints)
      return fail(B200MDM_EINVAL, "split target encoder: latent_dim %% target_joints != 0 (model/mdm.py:427)");
  }
  int dev = 0;
  CUDA_TRY(cudaGetDevice(&dev));
  cudaDeviceProp prop;
  CUDA_TRY(cudaGetDeviceProperties(&prop, dev));
  if (prop.major != 9 || prop.minor != 0) return fail(B200MDM_ECUDA, "sm_90a device required (found sm_%d%d)", prop.major, prop.minor);
  TRY(init_kernel_attrs());
  TRY(resolve_driver());
  b200mdm_engine* e = new b200mdm_engine();
  e->cfg = *cfg;
  e->d = cfg->latent_dim;
  e->ff = cfg->ff_size;
  e->L = cfg->num_layers;
  e->H = cfg->num_heads;
  e->JF = cfg->njoints * cfg->nfeats;
  e->Kp_in = (e->JF + 7) & ~7;
  e->N_out_pad = ((e->JF + 95) / 96) * 96;
  e->num_sms = prop.multiProcessorCount;
  e->layers.resize(e->L);
  e->dec = cfg->arch == B200MDM_ARCH_TRANS_DEC;
  e->dec_clip = e->dec && cfg->dec_memory == B200MDM_DEC_MEMORY_CLIP;
  e->ctx = e->dec ? cfg->context_len : 0;
  e->s_off = (e->dec && !e->dec_clip) ? e->ctx : 1;   // token 0: the encoder's conditioning / the decoder's timestep
  // DiP samples with guidance 7.5 (three times the encoder's 2.5): the CFG blend multiplies every activation rounding
  // error by ~10.  Its fp16 activations are therefore kept as hi + lo pairs; at 60-token sequences the doubled K of
  // the layer GEMMs is free.  The CLIP decoder runs 197-token sequences, where it is not, and holds the 1e-3 bound
  // with plain fp16 activations (DESIGN.md section 2).
  e->kw = (e->dec && !e->dec_clip) ? 2 : 1;
  CUDA_TRY(cudaStreamCreateWithFlags(&e->work, cudaStreamNonBlocking));
  CUDA_TRY(cudaEventCreateWithFlags(&e->ev_in, cudaEventDisableTiming));
  CUDA_TRY(cudaEventCreateWithFlags(&e->ev_out, cudaEventDisableTiming));
  TRY(dalloc(&e->state, 1, true));
  *out = e;
  return B200MDM_OK;
}

static void drop_graph(Workspace* w) {
  if (w->graph_exec) cudaGraphExecDestroy(w->graph_exec);
  w->graph_exec = nullptr;
  w->graph_key = GraphKey();
}
static void free_workspace(Workspace* w) {
  drop_graph(w);
  dfree(w->xin16); dfree(w->hres); dfree(w->qkv16); dfree(w->att16); dfree(w->ffn16); dfree(w->g16);
  dfree(w->tok0); dfree(w->condproj); dfree(w->proj); dfree(w->scale); dfree(w->x_work); dfree(w->pe_bias); dfree(w->eps_buf);
  dfree(w->kvlen); dfree(w->tvec); dfree(w->action); dfree(w->slots);
  dfree(w->encperm); dfree(w->memtok); dfree(w->memproj); dfree(w->mem16); dfree(w->qc16); dfree(w->kvc16); dfree(w->memmask);
  dfree(w->cross_mb); dfree(w->cross_u); dfree(w->cross_b); dfree(w->cross_c);
  dfree(w->tgt_valid); dfree(w->tgt_g); dfree(w->hs_desc); dfree(w->jg_x0); dfree(w->mp_x0);
  dfree(w->plms_ring); dfree(w->plms_mid); dfree(w->plms_pred);
  dfree(w->dpm_hist);
  dfree(w->vb_xs); dfree(w->vb_part); dfree(w->vb_terms);
  *w = Workspace();
}
// every workspace (the one in use and the parked ones): after a weight reload or a schedule-table move their graphs
// and derived tables (pe_bias, condproj, memproj) are stale
static void free_all_workspaces(b200mdm_engine* e) {
  free_workspace(static_cast<Workspace*>(e));
  for (auto& w : e->pool) free_workspace(&w);
  e->pool.clear();
}
static void drop_all_graphs(b200mdm_engine* e) {
  drop_graph(static_cast<Workspace*>(e));
  for (auto& w : e->pool) drop_graph(&w);
}

// the fp16 / packed copies b200mdm_finalize_weights derives from the weight store
static void free_repacks(b200mdm_engine* e) {
  for (auto& l : e->layers) { dfree(l.wqkv); dfree(l.wo); dfree(l.w1); dfree(l.w2); dfree(l.wq_c); dfree(l.wo_c); }
  dfree(e->w_in3); dfree(e->w_out3); dfree(e->temb_hidden); dfree(e->temb_table); dfree(e->wkv_all); dfree(e->bkv_all);
  dfree(e->cross_t);
}

extern "C" int b200mdm_destroy(b200mdm_engine* e) {
  if (!e) return B200MDM_OK;
  cudaDeviceSynchronize();
  free_all_workspaces(e);
  for (auto& kv : e->store) cudaFree(kv.second.dev);
  free_repacks(e);
  for (float*& t : e->tab) dfree(t);
  dfree(e->tmap);
  dfree(e->chain_mem); dfree(e->chain_mask); dfree(e->chain_prefix);
  dfree(e->goal_carry); dfree(e->goal_tgt);
  dfree(e->tw0); dfree(e->tb0); dfree(e->twk); dfree(e->tbk); dfree(e->twsum);
  dfree(e->state);
  dfree(e->jg_desc);
  dfree(e->ig_pairs);
  dfree(e->fg_len);
  dfree(e->pw_desc);
  if (e->work) cudaStreamDestroy(e->work);
  if (e->ev_in) cudaEventDestroy(e->ev_in);
  if (e->ev_out) cudaEventDestroy(e->ev_out);
  delete e;
  return B200MDM_OK;
}

// ------------------------------------------------------------------------------------------------ weights
static bool known_weight_name(const b200mdm_engine* e, const std::string& n) {
  static const char* fixed[] = {"input_process.poseEmbedding.weight", "input_process.poseEmbedding.bias",
                                "embed_timestep.time_embed.0.weight", "embed_timestep.time_embed.0.bias",
                                "embed_timestep.time_embed.2.weight", "embed_timestep.time_embed.2.bias",
                                "embed_text.weight", "embed_text.bias", "embed_action.action_embedding",
                                "output_process.poseFinal.weight", "output_process.poseFinal.bias",
                                "sequence_pos_encoder.pe", "embed_timestep.sequence_pos_encoder.pe"};
  for (const char* f : fixed)
    if (n == f) return true;
  static const char* per_layer[] = {"self_attn.in_proj_weight", "self_attn.in_proj_bias", "self_attn.out_proj.weight",
                                    "self_attn.out_proj.bias", "linear1.weight", "linear1.bias", "linear2.weight",
                                    "linear2.bias", "norm1.weight", "norm1.bias", "norm2.weight", "norm2.bias",
                                    "multihead_attn.in_proj_weight", "multihead_attn.in_proj_bias",
                                    "multihead_attn.out_proj.weight", "multihead_attn.out_proj.bias", "norm3.weight", "norm3.bias"};
  const std::string pre = e->dec ? "seqTransDecoder.layers." : "seqTransEncoder.layers.";
  if (n.compare(0, pre.size(), pre) == 0) {
    size_t dot = n.find('.', pre.size());
    if (dot == std::string::npos) return false;
    int l = atoi(n.substr(pre.size(), dot - pre.size()).c_str());
    if (l < 0 || l >= e->L) return false;
    std::string rest = n.substr(dot + 1);
    for (const char* f : per_layer)
      if (rest == f) return true;
  }
  if (e->cfg.target_encoder != B200MDM_TARGET_NONE) {
    const int tl = e->cfg.target_enc_layers, nj = e->cfg.target_joints;
    auto lin = [](const std::string& r, int max_layer) {   // "<2k>.weight" / "<2k>.bias", k = 0..max_layer
      for (int k = 0; k <= max_layer; ++k)
        if (r == std::to_string(2 * k) + ".weight" || r == std::to_string(2 * k) + ".bias") return true;
      return false;
    };
    auto joint = [nj](const std::string& r, std::string* tail) {   // "<i>.<tail>", i = 0..nj-1
      size_t dot = r.find('.');
      if (dot == std::string::npos || dot == 0 || r.find_first_not_of("0123456789") != dot) return false;
      if (atoi(r.substr(0, dot).c_str()) >= nj) return false;
      *tail = r.substr(dot + 1);
      return true;
    };
    const std::string pre = "embed_target_cond.";
    if (n.compare(0, pre.size(), pre) != 0) return false;
    const std::string r = n.substr(pre.size());
    std::string tail;
    switch (e->cfg.target_encoder) {
      case B200MDM_TARGET_SINGLE:
        return r.compare(0, 4, "mlp.") == 0 && lin(r.substr(4), tl);
      case B200MDM_TARGET_SPLIT:
        return r.compare(0, 10, "mini_mlps.") == 0 && joint(r.substr(10), &tail) && lin(tail, tl);
      case B200MDM_TARGET_MULTI:
        if (r == "target_all_loc_emb.weights") return true;
        return r.compare(0, 15, "target_loc_emb.") == 0 && joint(r.substr(15), &tail) && lin(tail, 1);
    }
  }
  return false;
}

extern "C" int b200mdm_load_weight(b200mdm_engine* e, const char* name, const float* data, const int64_t* shape,
                                   int32_t ndim) {
  if (!e || !name || !data || !shape || ndim < 1 || ndim > 4) return fail(B200MDM_EINVAL, "bad argument");
  std::string n(name);
  if (!known_weight_name(e, n)) return fail(B200MDM_EINVAL, "unexpected state_dict key '%s'", name);
  size_t numel = 1;
  std::vector<int64_t> shp(shape, shape + ndim);
  for (int64_t s : shp) {
    if (s <= 0) return fail(B200MDM_EINVAL, "bad shape for '%s'", name);
    numel *= static_cast<size_t>(s);
  }
  Tensor32& t = e->store[n];
  if (t.dev && t.numel != numel) { cudaFree(t.dev); t.dev = nullptr; }
  if (!t.dev) TRY(dalloc(&t.dev, numel));
  t.shape = shp;
  t.numel = numel;
  CUDA_TRY(cudaMemcpy(t.dev, data, numel * sizeof(float), cudaMemcpyDefault));
  e->finalized = false;
  return B200MDM_OK;
}

static int need(b200mdm_engine* e, const std::string& name, std::initializer_list<int64_t> shape, const float** out) {
  auto it = e->store.find(name);
  if (it == e->store.end()) return fail(B200MDM_ESTATE, "missing weight '%s'", name.c_str());
  std::vector<int64_t> want(shape);
  // allow a leading singleton / trailing squeeze for the positional table [max_len, 1, d]
  size_t numel = 1;
  for (int64_t s : want) numel *= static_cast<size_t>(s);
  if (it->second.numel != numel) return fail(B200MDM_EINVAL, "weight '%s' has %zu elements, expected %zu", name.c_str(), it->second.numel, numel);
  *out = it->second.dev;
  return B200MDM_OK;
}

static int to_f16(const float* src, __half** dst, size_t n, cudaStream_t s) {
  TRY(dalloc(dst, n));
  f32_to_f16_kernel<<<512, 256, 0, s>>>(src, *dst, n);
  CUDA_TRY(cudaGetLastError());
  return B200MDM_OK;
}
// W [N, K] -> fp16 [N, kw * K]: kw = 2 repeats W along K for activations kept as [hi | lo] (trans_dec engine)
static int to_f16_k(const float* src, __half** dst, int N, int K, int kw, cudaStream_t s) {
  if (kw == 1) return to_f16(src, dst, static_cast<size_t>(N) * K, s);
  TRY(dalloc(dst, static_cast<size_t>(N) * K * 2));
  f32_to_f16_dup_kernel<<<512, 256, 0, s>>>(src, *dst, N, K);
  CUDA_TRY(cudaGetLastError());
  return B200MDM_OK;
}

// embed_target_cond.* -> the packed layout of target_embed_kernel (kernels.cuh): w0 [G][dj][in], b0 [G][dj],
// wk [layers][G][dj][dj], bk [layers][G][dj], wsum [G] (multi).  nn.Linear weights are [out, in] already.
static int pack_target_weights(b200mdm_engine* e, cudaStream_t s) {
  dfree(e->tw0); dfree(e->tb0); dfree(e->twk); dfree(e->tbk); dfree(e->twsum);
  const int enc = e->cfg.target_encoder, n = e->cfg.target_joints, d = e->d;
  if (enc == B200MDM_TARGET_NONE) return B200MDM_OK;
  const bool multi = enc == B200MDM_TARGET_MULTI;
  e->tG = enc == B200MDM_TARGET_SINGLE ? 1 : n;
  e->tdj = enc == B200MDM_TARGET_SPLIT ? d / n : d;
  e->tin = enc == B200MDM_TARGET_SINGLE ? 4 * n : multi ? 3 : 4;
  e->tlayers = multi ? 1 : e->cfg.target_enc_layers;
  const int G = e->tG, dj = e->tdj, in = e->tin, L = e->tlayers;
  TRY(dalloc(&e->tw0, static_cast<size_t>(G) * dj * in));
  TRY(dalloc(&e->tb0, static_cast<size_t>(G) * dj));
  TRY(dalloc(&e->twk, static_cast<size_t>(L > 0 ? L : 1) * G * dj * dj));
  TRY(dalloc(&e->tbk, static_cast<size_t>(L > 0 ? L : 1) * G * dj));
  for (int i = 0; i < G; ++i) {
    const std::string p = enc == B200MDM_TARGET_SINGLE ? std::string("embed_target_cond.mlp.")
                          : multi ? "embed_target_cond.target_loc_emb." + std::to_string(i) + "."
                                  : "embed_target_cond.mini_mlps." + std::to_string(i) + ".";
    const float *w, *b;
    TRY(need(e, p + "0.weight", {dj, in}, &w));
    TRY(need(e, p + "0.bias", {dj}, &b));
    CUDA_TRY(cudaMemcpyAsync(e->tw0 + static_cast<size_t>(i) * dj * in, w, sizeof(float) * dj * in, cudaMemcpyDeviceToDevice, s));
    CUDA_TRY(cudaMemcpyAsync(e->tb0 + static_cast<size_t>(i) * dj, b, sizeof(float) * dj, cudaMemcpyDeviceToDevice, s));
    for (int l = 0; l < L; ++l) {
      const std::string k = std::to_string(2 * (l + 1));
      TRY(need(e, p + k + ".weight", {dj, dj}, &w));
      TRY(need(e, p + k + ".bias", {dj}, &b));
      CUDA_TRY(cudaMemcpyAsync(e->twk + (static_cast<size_t>(l) * G + i) * dj * dj, w, sizeof(float) * dj * dj,
                               cudaMemcpyDeviceToDevice, s));
      CUDA_TRY(cudaMemcpyAsync(e->tbk + (static_cast<size_t>(l) * G + i) * dj, b, sizeof(float) * dj, cudaMemcpyDeviceToDevice, s));
    }
  }
  if (multi) {
    const float* ws;
    TRY(need(e, "embed_target_cond.target_all_loc_emb.weights", {n}, &ws));
    TRY(dalloc(&e->twsum, n));
    CUDA_TRY(cudaMemcpyAsync(e->twsum, ws, sizeof(float) * n, cudaMemcpyDeviceToDevice, s));
  }
  return B200MDM_OK;
}

// g [B, d] = embed_target_cond(target [B, n, 3], valid_dev [B, n] fp32) on stream s
static int embed_target(b200mdm_engine* e, const float* target_dev, const float* valid_dev, int B, float* g_dev, cudaStream_t s) {
  const int n = e->cfg.target_joints, d = e->d;
  const size_t smem = sizeof(float) * (4 * n + 2 * d);
  target_embed_kernel<<<B, d, smem, s>>>(target_dev, valid_dev, e->tw0, e->tb0, e->twk, e->tbk, e->twsum, g_dev, n, e->tG,
                                         e->tdj, e->tin, e->tlayers, e->cfg.target_encoder == B200MDM_TARGET_MULTI ? 1 : 0);
  CUDA_TRY(cudaGetLastError());
  return B200MDM_OK;
}
// ... with the validity from the host: valid_dev receives it as fp32 (staged through `staging`, which must stay alive
// until the copy has run)
static int encode_target(b200mdm_engine* e, const float* target_dev, const uint8_t* valid_host, int B, float* valid_dev,
                         float* g_dev, std::vector<float>& staging, cudaStream_t s) {
  const int n = e->cfg.target_joints;
  staging.assign(static_cast<size_t>(B) * n, 0.f);
  for (size_t i = 0; i < staging.size(); ++i) staging[i] = valid_host[i] ? 1.f : 0.f;
  CUDA_TRY(cudaMemcpyAsync(valid_dev, staging.data(), staging.size() * sizeof(float), cudaMemcpyHostToDevice, s));
  return embed_target(e, target_dev, valid_dev, B, g_dev, s);
}

extern "C" int b200mdm_finalize_weights(b200mdm_engine* e, void* stream) {
  if (!e) return fail(B200MDM_EINVAL, "null engine");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int d = e->d, ff = e->ff, JF = e->JF;
  const float *w_in, *w_out, *t0w, *t0b, *t2w, *t2b;
  TRY(need(e, "input_process.poseEmbedding.weight", {d, JF}, &w_in));
  TRY(need(e, "input_process.poseEmbedding.bias", {d}, &e->b_in));
  TRY(need(e, "output_process.poseFinal.weight", {JF, d}, &w_out));
  TRY(need(e, "output_process.poseFinal.bias", {JF}, &e->b_out));
  TRY(need(e, "embed_timestep.time_embed.0.weight", {d, d}, &t0w));
  TRY(need(e, "embed_timestep.time_embed.0.bias", {d}, &t0b));
  TRY(need(e, "embed_timestep.time_embed.2.weight", {d, d}, &t2w));
  TRY(need(e, "embed_timestep.time_embed.2.bias", {d}, &t2b));
  TRY(need(e, "sequence_pos_encoder.pe", {e->cfg.pos_embed_max_len, d}, &e->pe));
  if (e->cfg.cond_mode == B200MDM_COND_TEXT) {
    TRY(need(e, "embed_text.weight", {d, e->cfg.cond_dim}, &e->w_txt));
    TRY(need(e, "embed_text.bias", {d}, &e->b_txt));
  } else if (e->cfg.cond_mode == B200MDM_COND_ACTION) {
    TRY(need(e, "embed_action.action_embedding", {e->cfg.num_actions, d}, &e->act_emb));
  }
  if (e->cfg.temb_rows > e->cfg.pos_embed_max_len) return fail(B200MDM_EINVAL, "temb_rows exceeds the positional table");

  // drop previous repacks; every workspace holds tables derived from the weights (pe_bias, condproj, memproj) and a
  // graph whose kernel parameters point at the old repacks: a forward that ran before this load must not leak into
  // the next one
  CUDA_TRY(cudaDeviceSynchronize());
  free_all_workspaces(e);
  free_repacks(e);

  // split-precision in / out projections: W' = [hi | hi | lo], zero padded
  const int Kp = e->Kp_in;
  TRY(dalloc(&e->w_in3, static_cast<size_t>(d) * 3 * Kp, true));
  split_weight_kernel<<<d, 128, 0, s>>>(w_in, e->w_in3, d, JF, Kp);
  CUDA_TRY(cudaGetLastError());
  TRY(dalloc(&e->w_out3, static_cast<size_t>(e->N_out_pad) * 3 * d, true));
  split_weight_kernel<<<JF, 128, 0, s>>>(w_out, e->w_out3, JF, d, d);
  CUDA_TRY(cudaGetLastError());
  TRY(make_map(&e->m_win, e->w_in3, d, 3 * Kp, 3 * Kp, 128));
  TRY(make_map(&e->m_wout, e->w_out3, e->N_out_pad, 3 * d, 3 * d, 96));

  for (int l = 0; l < e->L; ++l) {
    LayerW& w = e->layers[l];
    const std::string p = std::string(e->dec ? "seqTransDecoder.layers." : "seqTransEncoder.layers.") + std::to_string(l) + ".";
    const float *wqkv, *wo, *w1, *w2;
    TRY(need(e, p + "self_attn.in_proj_weight", {3 * d, d}, &wqkv));
    TRY(need(e, p + "self_attn.in_proj_bias", {3 * d}, &w.bqkv));
    TRY(need(e, p + "self_attn.out_proj.weight", {d, d}, &wo));
    TRY(need(e, p + "self_attn.out_proj.bias", {d}, &w.bo));
    TRY(need(e, p + "linear1.weight", {ff, d}, &w1));
    TRY(need(e, p + "linear1.bias", {ff}, &w.b1));
    TRY(need(e, p + "linear2.weight", {d, ff}, &w2));
    TRY(need(e, p + "linear2.bias", {d}, &w.b2));
    TRY(need(e, p + "norm1.weight", {d}, &w.g1));
    TRY(need(e, p + "norm1.bias", {d}, &w.be1));
    TRY(need(e, p + "norm2.weight", {d}, &w.g2));
    TRY(need(e, p + "norm2.bias", {d}, &w.be2));
    const int kw = e->kw;   // 2: weights repeated along K for [hi | lo] activations
    TRY(to_f16_k(wqkv, &w.wqkv, 3 * d, d, kw, s));
    TRY(to_f16_k(wo, &w.wo, d, d, kw, s));
    TRY(to_f16_k(w1, &w.w1, ff, d, kw, s));
    TRY(to_f16_k(w2, &w.w2, d, ff, kw, s));
    TRY(make_map(&w.m_wqkv, w.wqkv, 3 * d, kw * d, kw * d, 128));
    TRY(make_map(&w.m_w1, w.w1, ff, kw * d, kw * d, 128));
    TRY(make_map(&w.m_wo_256, w.wo, d, kw * d, kw * d, 256));
    TRY(make_map(&w.m_w2_256, w.w2, d, kw * ff, kw * ff, 256));
    if (e->dec) {
      // nn.MultiheadAttention in_proj rows: [Wq; Wk; Wv] -- query from the sequence, key/value from the text memory
      const float *wc, *bc, *woc;
      TRY(need(e, p + "multihead_attn.in_proj_weight", {3 * d, d}, &wc));
      TRY(need(e, p + "multihead_attn.in_proj_bias", {3 * d}, &bc));
      TRY(need(e, p + "multihead_attn.out_proj.weight", {d, d}, &woc));
      TRY(need(e, p + "multihead_attn.out_proj.bias", {d}, &w.bo_c));
      TRY(need(e, p + "norm3.weight", {d}, &w.g3));
      TRY(need(e, p + "norm3.bias", {d}, &w.be3));
      if (e->dec_clip) {   // one memory token: only the value rows and the output projection matter, in fp32
        w.wv_c32 = wc + static_cast<size_t>(2) * d * d;
        w.bv_c32 = bc + 2 * d;
        w.wo_c32 = woc;
        continue;
      }
      w.bq_c = bc;
      TRY(to_f16_k(wc, &w.wq_c, d, d, kw, s));
      if (l == 0) {
        TRY(dalloc(&e->wkv_all, static_cast<size_t>(e->L) * 2 * d * d));
        TRY(dalloc(&e->bkv_all, static_cast<size_t>(e->L) * 2 * d));
        TRY(make_map(&e->m_wkv_all, e->wkv_all, static_cast<uint64_t>(e->L) * 2 * d, d, d, 128));
      }
      f32_to_f16_kernel<<<512, 256, 0, s>>>(wc + static_cast<size_t>(d) * d, e->wkv_all + static_cast<size_t>(l) * 2 * d * d,
                                            static_cast<size_t>(2) * d * d);
      CUDA_TRY(cudaGetLastError());
      CUDA_TRY(cudaMemcpyAsync(e->bkv_all + static_cast<size_t>(l) * 2 * d, bc + d, sizeof(float) * 2 * d, cudaMemcpyDeviceToDevice, s));
      TRY(to_f16_k(woc, &w.wo_c, d, d, kw, s));
      TRY(make_map(&w.m_wq_c, w.wq_c, d, kw * d, kw * d, 128));
      TRY(make_map(&w.m_wo_c_256, w.wo_c, d, kw * d, kw * d, 256));
    }
  }
  // timestep-embedding MLP for every model timestep: temb[t] = W2 silu(W1 pe[t] + b1) + b2
  TRY(pack_target_weights(e, s));
  const int R = e->cfg.temb_rows;
  TRY(dalloc(&e->temb_hidden, static_cast<size_t>(R) * d));
  TRY(dalloc(&e->temb_table, static_cast<size_t>(R) * d));
  const size_t warps = static_cast<size_t>(R) * d;
  const int blocks = static_cast<int>((warps * 32 + 255) / 256);
  small_linear_kernel<1><<<blocks, 256, 0, s>>>(e->pe, t0w, t0b, e->temb_hidden, R, d, d, d);
  CUDA_TRY(cudaGetLastError());
  small_linear_kernel<0><<<blocks, 256, 0, s>>>(e->temb_hidden, t2w, t2b, e->temb_table, R, d, d, d);
  CUDA_TRY(cudaGetLastError());
  if (e->dec_clip) {
    // the timestep part of every layer's cross-attention row: cross_t[l, t] = W_o,l (W_v,l temb[t]) (temb_hidden is
    // free again and holds the inner product)
    TRY(dalloc(&e->cross_t, static_cast<size_t>(e->L) * R * d));
    for (int l = 0; l < e->L; ++l) {
      const LayerW& w = e->layers[l];
      small_linear_kernel<0><<<blocks, 256, 0, s>>>(e->temb_table, w.wv_c32, nullptr, e->temb_hidden, R, d, d, d);
      CUDA_TRY(cudaGetLastError());
      small_linear_kernel<0><<<blocks, 256, 0, s>>>(e->temb_hidden, w.wo_c32, nullptr, e->cross_t + static_cast<size_t>(l) * R * d,
                                                    R, d, d, d);
      CUDA_TRY(cudaGetLastError());
    }
  }
  CUDA_TRY(cudaStreamSynchronize(s));
  e->finalized = true;
  return B200MDM_OK;
}

// ------------------------------------------------------------------------------------------------ schedule
extern "C" int b200mdm_set_schedule(b200mdm_engine* e, int32_t n_steps, const float* rows_host,
                                    const int32_t* timestep_map_host) {
  if (!e || n_steps <= 0 || !rows_host || !timestep_map_host) return fail(B200MDM_EINVAL, "bad argument");
  for (int i = 0; i < n_steps; ++i)
    if (timestep_map_host[i] < 0 || timestep_map_host[i] >= e->cfg.temb_rows)
      return fail(B200MDM_EINVAL, "timestep_map[%d] = %d outside the pre-embedded range [0, %d)", i, timestep_map_host[i],
                  e->cfg.temb_rows);
  CUDA_TRY(cudaDeviceSynchronize());  // a loop still in flight may be reading the old tables
  if (n_steps > e->sched_cap) {
    // the captured step graphs hold these pointers as kernel parameters: moving the tables invalidates every graph
    drop_all_graphs(e);
    for (float*& t : e->tab) dfree(t);
    dfree(e->tmap);
    e->sched_cap = 0;
    const int cap = n_steps > 1000 ? n_steps : 1000;
    for (int t = 0; t < N_TABLES; ++t) TRY(dalloc(&e->tab[t], static_cast<size_t>(cap) * TAB_STRIDE[t]));
    TRY(dalloc(&e->tmap, cap));
    e->sched_cap = cap;
  }
  e->n_steps = n_steps;
  for (int t = 0; t < N_TABLES; ++t) e->tab_fresh[t] = t == TAB_STEP;
  CUDA_TRY(cudaMemcpy(e->tab[TAB_STEP], rows_host, static_cast<size_t>(n_steps) * SCHED_STRIDE * sizeof(float),
                      cudaMemcpyHostToDevice));
  CUDA_TRY(cudaMemcpy(e->tmap, timestep_map_host, static_cast<size_t>(n_steps) * sizeof(int), cudaMemcpyHostToDevice));
  return B200MDM_OK;
}

// The rows of table `which` for the current schedule (b200mdm_set_schedule_next / _dpm / _vb).
static int upload_table(b200mdm_engine* e, SchedTable which, int32_t n_steps, const float* rows_host) {
  if (!e || !rows_host) return fail(B200MDM_EINVAL, "bad argument");
  if (e->n_steps <= 0) return fail(B200MDM_ESTATE, "b200mdm_set_schedule has not been called");
  if (n_steps != e->n_steps)
    return fail(B200MDM_EINVAL, "n_steps %d differs from the schedule's %d", n_steps, e->n_steps);
  CUDA_TRY(cudaDeviceSynchronize());  // a loop still in flight may be reading the old rows
  CUDA_TRY(cudaMemcpy(e->tab[which], rows_host, static_cast<size_t>(n_steps) * TAB_STRIDE[which] * sizeof(float),
                      cudaMemcpyHostToDevice));
  e->tab_fresh[which] = true;
  return B200MDM_OK;
}
// ESTATE unless table `which` has been uploaded for the current schedule.
static int need_table(const b200mdm_engine* e, SchedTable which) {
  if (e->tab_fresh[which]) return B200MDM_OK;
  return fail(B200MDM_ESTATE, "%s has not been called for the current schedule", TAB_SETTER[which]);
}
// The output epilogue's pointer to each table.
static void set_tables(EpiOutParams* p, float* const (&tab)[N_TABLES]) {
  p->sched = tab[TAB_STEP];
  p->sched_next = tab[TAB_NEXT];
  p->sched_dpm = tab[TAB_DPM];
  p->sched_vb = tab[TAB_VB];
}

static_assert(MODE_X0 == B200MDM_MODE_X0 && MODE_DDPM == B200MDM_MODE_DDPM && MODE_DDIM == B200MDM_MODE_DDIM &&
                  MODE_DDIM_REVERSE == B200MDM_MODE_DDIM_REVERSE,
              "the output epilogue's modes are the public ones");
extern "C" int b200mdm_set_schedule_next(b200mdm_engine* e, int32_t n_steps, const float* rows_host) {
  return upload_table(e, TAB_NEXT, n_steps, rows_host);
}
extern "C" int b200mdm_set_schedule_dpm(b200mdm_engine* e, int32_t n_steps, const float* rows_host) {
  return upload_table(e, TAB_DPM, n_steps, rows_host);
}
extern "C" int b200mdm_set_schedule_vb(b200mdm_engine* e, int32_t n_steps, const float* rows_host) {
  return upload_table(e, TAB_VB, n_steps, rows_host);
}

// ------------------------------------------------------------------------------------------------ cond / workspace
static void attach_l2_window(b200mdm_engine* e, cudaStream_t stream = nullptr);

static int build_workspace(b200mdm_engine* e, int B, int T, int halves, int groups, cudaStream_t s) {
  const int d = e->d, S = T + e->s_off, Bp = (groups ? groups : halves) * B;
  const size_t g16_rows = static_cast<size_t>(groups ? Bp : B) * T;     // frame rows of the blend's output
  const int cond_rows = groups ? Bp - B : B;                             // rows of proj / action: the conditional ones
  const size_t M = static_cast<size_t>(Bp) * S, MB = static_cast<size_t>(B) * S;
  TRY(dalloc(&e->xin16, MB * 3 * e->Kp_in, true));
  const int kw = e->kw;
  TRY(dalloc(&e->hres, M * d * 2, true));   // residual stream, fp16 [hi | lo]
  TRY(dalloc(&e->qkv16, M * 3 * d));
  TRY(dalloc(&e->att16, M * d * kw));
  TRY(dalloc(&e->ffn16, M * e->ff * kw));
  TRY(dalloc(&e->g16, g16_rows * 3 * d));                              // frame rows only
  TRY(dalloc(&e->tok0, static_cast<size_t>(Bp) * d));
  TRY(dalloc(&e->condproj, static_cast<size_t>(Bp) * d, true));
  TRY(dalloc(&e->proj, static_cast<size_t>(cond_rows) * d, true));
  TRY(dalloc(&e->scale, B, true));
  TRY(dalloc(&e->x_work, static_cast<size_t>(B) * e->JF * T));
  TRY(dalloc(&e->kvlen, Bp));
  TRY(dalloc(&e->tvec, B, true));
  TRY(dalloc(&e->action, cond_rows, true));
  if (groups) TRY(dalloc(&e->mp_x0, static_cast<size_t>(Bp) * e->JF * T));
  if (e->dec_clip) {
    const size_t rows = static_cast<size_t>(Bp) * d, all = static_cast<size_t>(e->L) * Bp * d;
    TRY(dalloc(&e->cross_mb, rows));
    TRY(dalloc(&e->cross_u, rows));
    TRY(dalloc(&e->cross_b, all));
    TRY(dalloc(&e->cross_c, all));
  } else if (e->dec) {
    TRY(dalloc(&e->qc16, M * d));
    TRY(make_map_t(&e->m_qc_st, e->qc16, 2, M, d, d, 32));
    e->Mt = 0;              // the text-memory buffers are sized by the packed batch: b200mdm_set_cond_dec rebuilds them
    e->prefix_set = false;  // xin16 was reallocated
  }
  e->B = B; e->T = T; e->S = S; e->halves = halves; e->groups = groups; e->Bp = Bp;
  e->M = static_cast<int>(M); e->MB = static_cast<int>(MB);
  attach_l2_window(e);
  TRY(make_map(&e->m_xin, e->xin16, MB, 3 * e->Kp_in, 3 * e->Kp_in, GEMM_BLOCK_M));
  // GEMM A operand = the hi half of the residual stream (kw = 2, trans_dec: both halves, K = 2d against [W | W])
  TRY(make_map(&e->m_h16, e->hres, M, kw * d, 2 * d, GEMM_BLOCK_M));
  TRY(make_map(&e->m_att, e->att16, M, kw * d, kw * d, GEMM_BLOCK_M));
  TRY(make_map(&e->m_ffn, e->ffn16, M, kw * e->ff, kw * e->ff, GEMM_BLOCK_M));
  TRY(make_map(&e->m_g16, e->g16, g16_rows, 3 * d, 3 * d, GEMM_BLOCK_M));
  TRY(make_map_t(&e->m_qkv_st, e->qkv16, 2, M, 3 * d, 3 * d, 32));
  TRY(make_attention_kv_map(&e->m_qkv_kv, e->qkv16, Bp, S, 3 * d));
  TRY(make_map_t(&e->m_ffn_st, e->ffn16, 2, M, kw * e->ff, kw * e->ff, 32));
  TRY(make_map_res(&e->m_res_c, e->hres, MB, d));
  // the embedding GEMM's second copy of the frame rows: the unconditional half, or the last (unconditional) group
  const int last = groups ? groups - 1 : halves - 1;
  TRY(make_map_res(&e->m_res_u, e->hres + static_cast<size_t>(last) * MB * d * 2, MB, d));
  TRY(make_hres_map(&e->m_hres, e->hres, M));
  TRY(dalloc(&e->pe_bias, static_cast<size_t>(S) * d));
  pe_bias_kernel<<<S, 128, 0, s>>>(e->pe_bias, e->pe, e->b_in, S, d);   // on the caller's stream: ordered before any forward
  CUDA_TRY(cudaGetLastError());
  TRY(dalloc(&e->eps_buf, static_cast<size_t>(B) * e->JF * T));
  if (e->cfg.target_encoder != B200MDM_TARGET_NONE) {
    TRY(dalloc(&e->tgt_valid, static_cast<size_t>(B) * e->cfg.target_joints));
    TRY(dalloc(&e->tgt_g, static_cast<size_t>(B) * d));
  }
  return B200MDM_OK;
}

// Keep the residual stream resident in the L2 when it takes at most half of it: every residual + LayerNorm GEMM reads
// and rewrites it, and the other activations of the layer stream through between two of them.  A larger window crowds
// those out.  Measured on an H100 (50 MB L2, DESIGN §5) against no window: over a2m's 8 MB stream the loop ran 0.5 %
// faster, over DiP's 31.5 MB 16 % slower, over c2's 51.6 MB 5 % slower.  The window is attached to the engine stream,
// so every kernel captured into the step graph inherits it; a workspace above the limit clears it.  Best effort:
// failures are ignored.
static void attach_l2_window(b200mdm_engine* e, cudaStream_t stream) {
  cudaDeviceProp prop;
  int dev = 0;
  if (cudaGetDevice(&dev) == cudaSuccess && cudaGetDeviceProperties(&prop, dev) == cudaSuccess && prop.persistingL2CacheMaxSize > 0) {
    const size_t want = static_cast<size_t>(e->M) * e->d * 2 * sizeof(__half);
    cudaStreamAttrValue attr;
    memset(&attr, 0, sizeof(attr));   // num_bytes 0: no window
    if (2 * want <= static_cast<size_t>(prop.l2CacheSize)) {
      const size_t carve = want < static_cast<size_t>(prop.persistingL2CacheMaxSize) ? want : static_cast<size_t>(prop.persistingL2CacheMaxSize);
      cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, carve);
      attr.accessPolicyWindow.base_ptr = e->hres;
      attr.accessPolicyWindow.num_bytes = want < static_cast<size_t>(prop.accessPolicyMaxWindowSize) ? want : static_cast<size_t>(prop.accessPolicyMaxWindowSize);
      attr.accessPolicyWindow.hitRatio = want <= carve ? 1.0f : static_cast<float>(carve) / static_cast<float>(want);
      attr.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
      attr.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
    }
    cudaStreamSetAttribute(stream ? stream : e->work, cudaStreamAttributeAccessPolicyWindow, &attr);
    cudaGetLastError();
  }
}

// Make the workspace for (B, T, halves, groups) the current one: the one in use if it matches, else a parked one, else a
// new one (the least recently used of more than `MAX_PARKED` parked workspaces is freed).
static int select_workspace(b200mdm_engine* e, int B, int T, int halves, cudaStream_t s, int groups = 0) {
  constexpr size_t MAX_PARKED = 3;
  Workspace* cur = static_cast<Workspace*>(e);
  e->last_use = ++e->use_clock;
  if (cur->B == B && cur->T == T && cur->halves == halves && cur->groups == groups) return B200MDM_OK;
  if (cur->B > 0) {
    e->pool.push_back(*cur);
    *cur = Workspace();
  }
  for (size_t i = 0; i < e->pool.size(); ++i) {
    if (e->pool[i].B == B && e->pool[i].T == T && e->pool[i].halves == halves && e->pool[i].groups == groups) {
      *cur = e->pool[i];
      e->pool.erase(e->pool.begin() + i);
      cur->last_use = e->use_clock;
      cur->cond_set = false;      // the caller is about to set the conditioning of this loop
      cur->prefix_set = false;
      cur->target_set = false;
      attach_l2_window(e);
      return B200MDM_OK;
    }
  }
  while (e->pool.size() > MAX_PARKED) {
    size_t lru = 0;
    for (size_t i = 1; i < e->pool.size(); ++i)
      if (e->pool[i].last_use < e->pool[lru].last_use) lru = i;
    CUDA_TRY(cudaDeviceSynchronize());   // a loop on that workspace may still be running
    free_workspace(&e->pool[lru]);
    e->pool.erase(e->pool.begin() + lru);
  }
  int r = build_workspace(e, B, T, halves, groups, s);
  if (r != B200MDM_OK) free_workspace(cur);
  cur->last_use = e->use_clock;
  return r;
}

// ---- the conditioning of one loop (set_conditioning, behind every b200mdm_set_cond*)
// a sequence of n_tokens tokens fits the positional table and the attention kernels
static int check_seq_len(const b200mdm_engine* e, int n_tokens) {
  if (n_tokens > e->cfg.pos_embed_max_len) return fail(B200MDM_EINVAL, "sequence longer than the positional table");
  if (n_tokens > ATC_MAX_KEYS)
    return fail(B200MDM_ENOTIMPL, "sequences of more than %d tokens (the attention kernels keep all keys of a sample on chip; "
                "every dataset of the reference stops at 196 frames)", ATC_MAX_KEYS);
  return B200MDM_OK;
}
// Valid-key counts of the current workspace's packed batch -- the seq_extra tokens ahead of the frames are always valid,
// then `lengths` frames (model/mdm.py:241-247; lengths_to_mask, data_loaders/tensors.py:3-6), all keys unless `clamp` --
// and the guidance scales, uploaded on s.  The host staging lives in the engine until the next call, so the asynchronous
// copy needs no stream synchronisation.
static int upload_kvlen_scale(b200mdm_engine* e, int nframes, int seq_extra, bool clamp, const int64_t* lengths_host,
                              const float* scale_dev, cudaStream_t s) {
  std::vector<int>& kv = e->h_kv;
  kv.assign(e->Bp, e->S);
  if (e->cfg.mask_frames && lengths_host && clamp) {
    for (int b = 0; b < e->Bp; ++b) {
      long long len = lengths_host[b % e->B];
      if (len < 0) len = 0;
      if (len > nframes) len = nframes;
      kv[b] = static_cast<int>(len) + seq_extra;
    }
  }
  CUDA_TRY(cudaMemcpyAsync(e->kvlen, kv.data(), kv.size() * sizeof(int), cudaMemcpyHostToDevice, s));
  if (scale_dev) CUDA_TRY(cudaMemcpyAsync(e->scale, scale_dev, e->B * sizeof(float), cudaMemcpyDeviceToDevice, s));
  return B200MDM_OK;
}
// condproj rows of the packed batch: proj = embed_text(text) [rows, d] when the model is text-conditioned and a text is
// given (model/mdm.py:218), then the conditional / unconditional rows of the model's conditioning mode
// (condproj_fill_kernel).  The rows = K * batch conditional rows (text_dev [K, batch, C], action [K * batch]) come first.
// slot >= 0 (b200mdm_slot_admit): text_dev is that one row's text, projected into proj row `slot`; every condproj row
// is then refilled from proj as it is, which rewrites the other rows with their own bits.
static int fill_condproj(b200mdm_engine* e, const float* text_dev, bool uncond, int rows, cudaStream_t s, int slot = -1) {
  const int d = e->d;
  if (e->cfg.cond_mode == B200MDM_COND_TEXT && text_dev) {
    const int n = slot >= 0 ? 1 : rows;
    const size_t warps = static_cast<size_t>(n) * d;
    small_linear_kernel<0><<<static_cast<int>((warps * 32 + 255) / 256), 256, 0, s>>>(
        text_dev, e->w_txt, e->b_txt, e->proj + static_cast<size_t>(slot >= 0 ? slot : 0) * d, n, d, e->cfg.cond_dim,
        e->cfg.cond_dim);
    CUDA_TRY(cudaGetLastError());
    e->launches++;
  }
  condproj_fill_kernel<<<e->Bp, 128, 0, s>>>(e->condproj, e->proj, e->b_txt, e->act_emb, e->action, rows, d, e->Bp,
                                             uncond ? 1 : 0, e->cfg.cond_mode);
  CUDA_TRY(cudaGetLastError());
  e->launches++;
  return B200MDM_OK;
}
// a new loop's conditioning is in place: the previous loop's target and inpainting inputs no longer apply
static void end_cond(b200mdm_engine* e) {
  e->cond_set = true;
  e->target_set = false;
  e->inpaint_mask = nullptr;
  e->inpaint_weight = nullptr;
  e->inpaint_motion = nullptr;
  e->hs_set = false;
  e->guide_terms = 0;
  e->pw_set = false;
  e->vb_live = false;
  e->chain_next = -1;
  e->slot_mode = false;
}

// cb_l[b']= W_o,l (W_v,l mb[b'] + b_v,l) + b_o,l with mb = condproj (+ g): the per-sample part of the cross-attention rows
// of a CLIP-memory decoder, once per loop (kernels.cuh, cross_rows_kernel).
static int cross_rows_per_sample(b200mdm_engine* e, const float* g, cudaStream_t s) {
  const int d = e->d, Bp = e->Bp;
  cross_mem_kernel<<<Bp, 128, 0, s>>>(e->cross_mb, e->condproj, g, e->B, d);
  CUDA_TRY(cudaGetLastError());
  const int blocks = static_cast<int>((static_cast<size_t>(Bp) * d * 32 + 255) / 256);
  for (int l = 0; l < e->L; ++l) {
    const LayerW& w = e->layers[l];
    small_linear_kernel<0><<<blocks, 256, 0, s>>>(e->cross_mb, w.wv_c32, w.bv_c32, e->cross_u, Bp, d, d, d);
    CUDA_TRY(cudaGetLastError());
    small_linear_kernel<0><<<blocks, 256, 0, s>>>(e->cross_u, w.wo_c32, w.bo_c, e->cross_b + static_cast<size_t>(l) * Bp * d,
                                                  Bp, d, d, d);
    CUDA_TRY(cudaGetLastError());
  }
  e->launches += 1 + 2 * e->L;
  return B200MDM_OK;
}

// trans_dec with a BERT memory and context_len > 0: DiP, the prefix-completion decoder (context_len 0 is the plain BERT
// decoder, which takes every sampling extension)
static bool is_prefix_engine(const b200mdm_engine* e) { return e->dec && !e->dec_clip && e->ctx > 0; }

// The text-memory buffers of the current workspace for Mt tokens, rebuilt when Mt changes: the projected prompt rows
// (B, or K * B under multi-prompt guidance) and the packed batch's Bp rows.
static int ensure_text_memory(b200mdm_engine* e, int Mt) {
  if (Mt == e->Mt) return B200MDM_OK;
  const int d = e->d, Bp = e->Bp, C = e->cfg.cond_dim;
  const size_t cond_rows = static_cast<size_t>(e->groups ? Bp - e->B : e->B);
  CUDA_TRY(cudaDeviceSynchronize());
  drop_graph(e);
  dfree(e->encperm); dfree(e->memtok); dfree(e->memproj); dfree(e->mem16); dfree(e->kvc16); dfree(e->memmask);
  e->Mt = 0;   // until every buffer below exists: a failed allocation leaves the next call to rebuild them
  TRY(dalloc(&e->encperm, cond_rows * Mt * C));
  TRY(dalloc(&e->memtok, cond_rows * Mt * d));
  TRY(dalloc(&e->memproj, static_cast<size_t>(Bp) * Mt * d));
  TRY(dalloc(&e->mem16, static_cast<size_t>(Bp) * Mt * 2 * d));   // [hi | lo]
  TRY(dalloc(&e->kvc16, static_cast<size_t>(Bp) * Mt * 2 * d * e->L));      // [Bp*Mt, L * (k | v)]
  TRY(dalloc(&e->memmask, static_cast<size_t>(Bp) * Mt));
  TRY(make_map(&e->m_mem, e->mem16, static_cast<uint64_t>(Bp) * Mt, 2 * d, 2 * d, GEMM_BLOCK_M));
  TRY(make_map_t(&e->m_kvc_st, e->kvc16, 2, static_cast<uint64_t>(Bp) * Mt, 2 * d * e->L, 2 * d * e->L, 32));
  e->Mt = Mt;
  return B200MDM_OK;
}

// The padding mask [Bp, Mt] of a token memory over the packed batch of B samples, into dst: the K * B prompt rows are
// mask [K, B, Mt] as it is (group-major, the packed order); each unconditional row pads where every prompt pads for its
// sample, so it admits every token some prompt admits.  With K = 1 that is the sample's own mask, as in a classifier-free
// pair, and it does not depend on the prompts' order.  (The unconditional tokens are all equal, so any mask admitting
// one gives the same output up to rounding.)
static void pack_text_mask(unsigned char* dst, const uint8_t* mask, int K, int B, int Bp, int Mt) {
  const int rows = K * B;
  std::fill(dst, dst + static_cast<size_t>(Bp) * Mt, 1);
  for (int bp = 0; bp < rows; ++bp)
    for (int m = 0; m < Mt; ++m) {
      const unsigned char pad = mask[static_cast<size_t>(bp) * Mt + m] ? 1 : 0;
      dst[static_cast<size_t>(bp) * Mt + m] = pad;
      if (Bp > rows) dst[static_cast<size_t>(rows + bp % B) * Mt + m] &= pad;
    }
}

// The projected token memory [Bp * Mt, d] of the current workspace into dst, text_emb = embed_text(mask_cond(tokens))
// per token (model/mdm.py:218): W tokens + b for the K * B prompt rows (tokens [K, Mt, B, C], the reference layout per
// prompt), b for the unconditional rows, and b for every row with `uncond`.  K + 2 launches on s.
static int build_text_memory(b200mdm_engine* e, const float* tokens, int K, bool uncond, float* dst, cudaStream_t s) {
  const int d = e->d, B = e->B, Mt = e->Mt, C = e->cfg.cond_dim, rows = K * B;
  for (int k = 0; k < K; ++k) {
    permute_mbc_kernel<<<dim3(Mt, B), 128, 0, s>>>(tokens + static_cast<size_t>(k) * Mt * B * C,
                                                    e->encperm + static_cast<size_t>(k) * B * Mt * C, Mt, B, C);
    CUDA_TRY(cudaGetLastError());
  }
  const size_t warps = static_cast<size_t>(rows) * Mt * d;
  small_linear_kernel<0><<<static_cast<int>((warps * 32 + 255) / 256), 256, 0, s>>>(e->encperm, e->w_txt, e->b_txt, e->memtok,
                                                                                     rows * Mt, d, C, C);
  CUDA_TRY(cudaGetLastError());
  memproj_group_fill_kernel<<<dim3(Mt, e->Bp), 128, 0, s>>>(dst, e->memtok, e->b_txt, uncond ? 0 : rows, Mt, d);
  CUDA_TRY(cudaGetLastError());
  e->launches += K + 2;
  return B200MDM_OK;
}

// ---- features that exclude each other or a sampler family.  The engine's twin of _REFUSED in
// diffusion/gaussian_diffusion.py, with the same sampler rows; the setter rows make handshakes, joint-position control
// and multi-prompt guidance pairwise exclusive and keep each off prefix-completion (DiP) engines.
enum Feature : unsigned { F_PREFIX = 1, F_HANDSHAKE = 2, F_JOINT = 4, F_MULTI = 8, F_TOKENS = 16, F_TARGET = 32, F_INPAINT = 64 };
enum Family { FAM_REVERSE, FAM_PLMS, FAM_DPM, FAM_VB, FAM_HANDSHAKE, FAM_JOINT, FAM_MULTI, FAM_SLOTS, FAM_STEP_AT };
static const struct {
  const char* name;
  unsigned refuses;
} REFUSED[] = {
    {"DDIM inversion", F_HANDSHAKE | F_JOINT},
    {"PLMS", F_JOINT},
    {"DPM-Solver++", F_JOINT},
    {"the variational bound", F_HANDSHAKE | F_JOINT | F_MULTI},
    {"handshaking", F_PREFIX | F_JOINT | F_MULTI},
    {"joint-position control", F_PREFIX | F_HANDSHAKE | F_MULTI},
    {"multi-prompt guidance", F_PREFIX},
    // a schedule index per row: every per-loop input but the conditioning rows or token memory, prefix, scale and
    // lengths is one for the batch (a token memory and a prefix are per slot in a b200mdm_chain_slots_begin session)
    {"continuous batching", F_HANDSHAKE | F_JOINT | F_MULTI | F_TARGET | F_INPAINT},
    // b200mdm_sample_step_at: the rows of the one conditioning upload, so no token memory or prefix
    {"continuous batching", F_PREFIX | F_HANDSHAKE | F_JOINT | F_MULTI | F_TOKENS | F_TARGET | F_INPAINT},
};

// ENOTIMPL when the engine holds a feature (of those in `among`) that `family` refuses
static int refuse(const b200mdm_engine* e, Family family, unsigned among = ~0u) {
  static const char* const feature[] = {"prefix-completion (DiP) models", "handshakes", "joint-position control",
                                        "multi-prompt guidance", "BERT text memories", "target conditioning", "inpainting"};
  const unsigned live = (is_prefix_engine(e) ? F_PREFIX : 0u) | (e->hs_set ? F_HANDSHAKE : 0u) | (e->guide_terms ? F_JOINT : 0u) |
                        (e->groups ? F_MULTI : 0u) | (e->dec && !e->dec_clip ? F_TOKENS : 0u) |
                        (e->target_set ? F_TARGET : 0u) | (e->inpaint_mask || e->inpaint_weight ? F_INPAINT : 0u);
  const unsigned hit = REFUSED[family].refuses & among & live;
  for (int i = 0; i < 7; ++i)
    if (hit & (1u << i)) return fail(B200MDM_ENOTIMPL, "%s with %s is not implemented", REFUSED[family].name, feature[i]);
  return B200MDM_OK;
}

// What a b200mdm_set_cond* call hands to set_conditioning.  For everything the upload writes, the classifier-free batch
// (halves 1, or 2 with a scale) is the multi-prompt layout with K = 1; the two differ in the workspace's layout only.
struct CondIn {
  int batch, nframes;
  const int64_t* lengths;         // [batch] host, nullable
  const float* embed;             // text or CLIP rows [K, batch, C], or BERT token features [K, n_tokens, batch, C]
  int K = 1;
  bool multi = false;             // multi-prompt groups (G = K + 1), else classifier-free halves
  const uint8_t* mask = nullptr;  // [K, batch, n_tokens] host, 1 = padding (the CLIP row: [batch], all zero)
  int n_tokens = 0;
  const int64_t* action = nullptr;   // [batch, K] host
  const float* scale = nullptr;      // [batch] device: classifier-free guidance
  bool force_uncond = false;
};

// The conditioning of a loop: argument checks (all before any CUDA call), the workspace of the packed batch, its key
// counts and guidance scales, then the rows of the model family -- condproj rows (encoder; CLIP-memory decoder, with its
// per-sample cross-attention rows) or the token memory and its mask (BERT-memory decoder).
static int set_conditioning(b200mdm_engine* e, const CondIn& c, cudaStream_t s) {
  if (!e->finalized) return fail(B200MDM_ESTATE, "weights not finalised");
  if (c.batch <= 0 || c.nframes <= 0) return fail(B200MDM_EINVAL, "bad batch / nframes");
  if (c.K < 1 || c.K > MP_MAX_PROMPTS) return fail(B200MDM_EINVAL, "prompt count %d outside 1 .. %d", c.K, MP_MAX_PROMPTS);
  const bool bert = e->dec && !e->dec_clip;
  const int halves = c.scale ? 2 : 1, B = c.batch, rows = c.K * B, mode = e->cfg.cond_mode;
  const bool uncond = halves == 1 && c.force_uncond;
  if (bert) {
    if (c.n_tokens <= 0 || c.n_tokens > XAL_MAX_MT)
      return fail(B200MDM_EINVAL, "n_tokens %d: a text memory holds 1..%d tokens (DistilBERT's position limit)", c.n_tokens,
                  XAL_MAX_MT);
    if (!c.embed || !c.mask) return fail(B200MDM_EINVAL, "the BERT decoder needs the token features and their masks");
  } else if (e->dec_clip) {
    // y['text_embed'] [1, B, C] is the one memory token of every sample, without a padding mask (model/mdm.py:262-263)
    if (!c.multi && c.n_tokens != 1)
      return fail(B200MDM_EINVAL, "a CLIP-memory decoder takes one memory token per sample (n_tokens %d)", c.n_tokens);
    if (!c.embed || (!c.multi && !c.mask))
      return fail(B200MDM_EINVAL, "the CLIP decoder needs y['text_embed'] and an all-zero mask");
    for (int b = 0; !c.multi && b < B; ++b)
      if (c.mask[b]) return fail(B200MDM_EINVAL, "the CLIP memory has no padding mask (model/mdm.py:262-263)");
  } else {
    if (mode == B200MDM_COND_NONE && (c.multi || halves == 2))
      return fail(B200MDM_EINVAL, "%s needs a conditioned model (sampler_util.py:29)",
                  c.multi ? "multi-prompt guidance" : "classifier-free guidance");
    if (mode == B200MDM_COND_TEXT && !c.embed && !uncond)
      return fail(B200MDM_EINVAL, "text-conditioned model needs the text embeddings");
    if (mode == B200MDM_COND_ACTION && !c.action && !uncond)
      return fail(B200MDM_EINVAL, "action-conditioned model needs the actions");
  }
  TRY(check_seq_len(e, c.nframes + (bert ? e->ctx : 1)));
  std::vector<int>& a = e->h_action;
  const bool actions = mode == B200MDM_COND_ACTION && c.action;
  if (actions) {
    a.assign(rows, 0);
    for (int b = 0; b < B; ++b)
      for (int k = 0; k < c.K; ++k) {
        const int64_t v = c.action[static_cast<size_t>(b) * c.K + k];
        if (v < 0 || v >= e->cfg.num_actions) return fail(B200MDM_EINVAL, "action index out of range");
        a[static_cast<size_t>(k) * B + b] = static_cast<int>(v);   // group-major, as the packed batch
      }
  }
  TRY(select_workspace(e, B, c.nframes, halves, s, c.multi ? c.K + 1 : 0));
  if (bert) TRY(ensure_text_memory(e, c.n_tokens));
  // valid keys: the timestep token (the False column prepended, model/mdm.py:241-247) or DiP's context frames
  // (model/mdm.py:204-206), then `lengths` frames
  TRY(upload_kvlen_scale(e, c.nframes, bert ? e->ctx : 1, bert ? e->S > 1 : c.nframes > 1, c.lengths, c.scale, s));
  if (bert) {
    e->h_mask.resize(static_cast<size_t>(e->Bp) * e->Mt);
    pack_text_mask(e->h_mask.data(), c.mask, c.K, B, e->Bp, e->Mt);
    CUDA_TRY(cudaMemcpyAsync(e->memmask, e->h_mask.data(), e->h_mask.size(), cudaMemcpyHostToDevice, s));
    e->mem_uncond = uncond;
    TRY(build_text_memory(e, c.embed, c.K, uncond, e->memproj, s));
  } else {
    if (actions) CUDA_TRY(cudaMemcpyAsync(e->action, a.data(), a.size() * sizeof(int), cudaMemcpyHostToDevice, s));
    TRY(fill_condproj(e, c.embed, uncond, rows, s));
    if (e->dec_clip) TRY(cross_rows_per_sample(e, nullptr, s));
  }
  end_cond(e);
  return B200MDM_OK;
}

extern "C" int b200mdm_set_cond(b200mdm_engine* e, int32_t batch, int32_t nframes, const float* cond_embed_dev,
                                const int64_t* lengths_host, const float* scale_dev, int32_t force_uncond,
                                const int64_t* action_host, void* stream) {
  if (!e) return fail(B200MDM_EINVAL, "null engine");
  if (e->dec) return fail(B200MDM_EINVAL, "trans_dec engines take their conditioning through b200mdm_set_cond_dec");
  CondIn c{batch, nframes, lengths_host, cond_embed_dev};
  c.action = action_host;
  c.scale = scale_dev;
  c.force_uncond = force_uncond != 0;
  return set_conditioning(e, c, static_cast<cudaStream_t>(stream));
}

// trans_dec: the BERT token features + padding mask (DiP, and the plain BERT decoder), or the CLIP row
extern "C" int b200mdm_set_cond_dec(b200mdm_engine* e, int32_t batch, int32_t nframes, const float* enc_text_dev,
                                    const uint8_t* text_mask_host, int32_t n_tokens, const int64_t* lengths_host,
                                    const float* scale_dev, int32_t force_uncond, void* stream) {
  if (!e) return fail(B200MDM_EINVAL, "null engine");
  if (!e->dec) return fail(B200MDM_EINVAL, "b200mdm_set_cond_dec is for trans_dec engines");
  CondIn c{batch, nframes, lengths_host, enc_text_dev};
  c.mask = text_mask_host;
  c.n_tokens = n_tokens;
  c.scale = scale_dev;
  c.force_uncond = force_uncond != 0;
  return set_conditioning(e, c, static_cast<cudaStream_t>(stream));
}

// ---- multi-prompt guidance (DESIGN.md, "Multi-prompt guidance")
extern "C" int b200mdm_set_cond_multi(b200mdm_engine* e, int32_t batch, int32_t nframes, int32_t K,
                                      const float* prompt_embed_dev, const int64_t* lengths_host,
                                      const int64_t* prompt_action_host, void* stream) {
  if (!e) return fail(B200MDM_EINVAL, "null engine");
  if (e->dec) return fail(B200MDM_EINVAL, "trans_dec engines take their prompts through b200mdm_set_cond_multi_dec");
  CondIn c{batch, nframes, lengths_host, prompt_embed_dev, K, true};
  c.action = prompt_action_host;
  return set_conditioning(e, c, static_cast<cudaStream_t>(stream));
}

extern "C" int b200mdm_set_cond_multi_dec(b200mdm_engine* e, int32_t batch, int32_t nframes, int32_t K,
                                          const float* prompt_clip_dev, const int64_t* lengths_host, void* stream) {
  if (!e) return fail(B200MDM_EINVAL, "null engine");
  if (!e->dec) return fail(B200MDM_EINVAL, "b200mdm_set_cond_multi_dec is for trans_dec engines");
  TRY(refuse(e, FAM_MULTI));
  if (!e->dec_clip)
    return fail(B200MDM_EINVAL, "BERT-memory decoders take their prompts through b200mdm_set_cond_multi_tokens");
  return set_conditioning(e, CondIn{batch, nframes, lengths_host, prompt_clip_dev, K, true}, static_cast<cudaStream_t>(stream));
}

extern "C" int b200mdm_set_cond_multi_tokens(b200mdm_engine* e, int32_t batch, int32_t nframes, int32_t K,
                                             const float* tokens_dev, const uint8_t* mask_host, int32_t n_tokens,
                                             const int64_t* lengths_host, void* stream) {
  if (!e) return fail(B200MDM_EINVAL, "null engine");
  if (!e->dec) return fail(B200MDM_EINVAL, "b200mdm_set_cond_multi_tokens is for trans_dec engines");
  TRY(refuse(e, FAM_MULTI));
  if (e->dec_clip) return fail(B200MDM_EINVAL, "CLIP-memory decoders take their prompts through b200mdm_set_cond_multi_dec");
  CondIn c{batch, nframes, lengths_host, tokens_dev, K, true};
  c.mask = mask_host;
  c.n_tokens = n_tokens;
  return set_conditioning(e, c, static_cast<cudaStream_t>(stream));
}

extern "C" int b200mdm_set_target(b200mdm_engine* e, const float* target_dev, const uint8_t* valid_host, void* stream) {
  if (!e || !target_dev || !valid_host) return fail(B200MDM_EINVAL, "null argument");
  if (e->cfg.target_encoder == B200MDM_TARGET_NONE) return fail(B200MDM_EINVAL, "this engine has no target encoder");
  if (!e->cond_set) return fail(B200MDM_ESTATE, "call b200mdm_set_cond / b200mdm_set_cond_dec first (they size the workspace)");
  TRY(encode_target(e, target_dev, valid_host, e->B, e->tgt_valid, e->tgt_g, e->h_valid, static_cast<cudaStream_t>(stream)));
  e->launches++;
  // the CLIP decoder's memory row carries g as well (model/mdm.py:199,262): its per-sample cross-attention part again
  if (e->dec_clip) TRY(cross_rows_per_sample(e, e->tgt_g, static_cast<cudaStream_t>(stream)));
  e->target_set = true;
  return B200MDM_OK;
}

// y['prefix'] [B, J, F, context_len] (model/mdm.py:203-206): packed once per loop into the first context_len rows of
// every sequence of the embedding GEMM's A operand.
extern "C" int b200mdm_set_prefix(b200mdm_engine* e, const float* prefix_dev, void* stream) {
  if (!e || !prefix_dev) return fail(B200MDM_EINVAL, "null argument");
  if (!e->dec || e->ctx <= 0) return fail(B200MDM_EINVAL, "this engine has no prefix (context_len == 0)");
  if (!e->cond_set) return fail(B200MDM_ESTATE, "call b200mdm_set_cond_dec first (it sizes the workspace)");
  TRY(launch_pack_input(prefix_dev, e->xin16, e->B, e->JF, e->ctx, e->S, e->Kp_in, 0, static_cast<cudaStream_t>(stream)));
  e->launches++;
  e->prefix_set = true;
  e->prefix_src = prefix_dev;
  e->chain_next = -1;   // a chain's prefix rows were replaced
  return B200MDM_OK;
}

extern "C" int b200mdm_set_inpaint(b200mdm_engine* e, const uint8_t* mask_dev, const float* motion_dev) {
  if (!e) return fail(B200MDM_EINVAL, "null engine");
  if ((mask_dev == nullptr) != (motion_dev == nullptr)) return fail(B200MDM_EINVAL, "inpainting needs both mask and motion");
  e->inpaint_mask = mask_dev;
  e->inpaint_weight = nullptr;
  e->inpaint_motion = motion_dev;
  return B200MDM_OK;
}

extern "C" int b200mdm_set_inpaint_weight(b200mdm_engine* e, const float* weight_dev, const float* motion_dev) {
  if (!e) return fail(B200MDM_EINVAL, "null engine");
  if ((weight_dev == nullptr) != (motion_dev == nullptr)) return fail(B200MDM_EINVAL, "soft inpainting needs both weight and motion");
  e->inpaint_mask = nullptr;
  e->inpaint_weight = weight_dev;
  e->inpaint_motion = motion_dev;
  return B200MDM_OK;
}

extern "C" int b200mdm_set_handshake(b200mdm_engine* e, int32_t h, const int64_t* lengths_host,
                                     const uint8_t* motion_start_host, void* stream) {
  if (!e) return fail(B200MDM_EINVAL, "null engine");
  if (h < 0) return fail(B200MDM_EINVAL, "handshake size %d < 0", h);
  TRY(refuse(e, FAM_HANDSHAKE, F_PREFIX));
  if (!e->cond_set) return fail(B200MDM_ESTATE, "call b200mdm_set_cond / b200mdm_set_cond_dec first (they size the workspace)");
  TRY(refuse(e, FAM_HANDSHAKE));
  TRY(handshake_desc(h, e->B, e->T, lengths_host, motion_start_host, &e->h_hs));
  e->hs_set = false;
  if (e->h_hs.empty()) return B200MDM_OK;   // nothing to blend: the plain forward
  if (!e->hs_desc) TRY(dalloc(&e->hs_desc, e->h_hs.size()));
  // the host staging lives in the engine until the next call (as b200mdm_set_cond's): no stream synchronisation
  CUDA_TRY(cudaMemcpyAsync(e->hs_desc, e->h_hs.data(), e->h_hs.size() * sizeof(int), cudaMemcpyHostToDevice,
                           static_cast<cudaStream_t>(stream)));
  e->hs_set = true;
  return B200MDM_OK;
}

// The argument checks of each term of joint-position control, shared by its setter and its test hook: each fills its
// part of a GuideDesc.  The joint terms:
static int fill_joint(const float* mean_dev, const float* std_dev, const float* target_dev, const float* weight_dev,
                      float step, int32_t iters, JointGuide* out) {
  if (!mean_dev || !std_dev || !target_dev || !weight_dev) return fail(B200MDM_EINVAL, "null argument");
  if (!std::isfinite(step) || step <= 0.f) return fail(B200MDM_EINVAL, "guidance step %g: a finite value > 0", step);
  if (iters < 1 || iters > 10000) return fail(B200MDM_EINVAL, "guidance iterations %d outside 1 .. 10000", iters);
  *out = JointGuide{mean_dev, std_dev, target_dev, weight_dev, step, iters};
  return B200MDM_OK;
}

// the foot terms, with lengths_host clamped to T in `len` (empty without lengths; the caller points out->lengths at them)
static int fill_foot(float contact_weight, float floor_weight, float floor_height, const float* contact_dev,
                     const int64_t* lengths_host, int B, int T, FootGuide* out, std::vector<int>* len) {
  if (!std::isfinite(contact_weight) || contact_weight < 0.f || !std::isfinite(floor_weight) || floor_weight < 0.f)
    return fail(B200MDM_EINVAL, "foot guidance weights %g, %g: finite values >= 0", contact_weight, floor_weight);
  if (!std::isfinite(floor_height)) return fail(B200MDM_EINVAL, "floor height %g: a finite value", floor_height);
  len->clear();
  for (int b = 0; lengths_host && b < B; ++b) {
    if (lengths_host[b] < 0) return fail(B200MDM_EINVAL, "lengths[%d] = %lld < 0", b, static_cast<long long>(lengths_host[b]));
    len->push_back(static_cast<int>(std::min<int64_t>(lengths_host[b], T)));
  }
  *out = FootGuide{contact_dev, nullptr, contact_weight, floor_weight, floor_height};
  return B200MDM_OK;
}

// one grid of the scene terms (NULL: no grid)
static int check_grid(const b200mdm_grid* g, const char* what, int B, SceneGrid* out) {
  *out = SceneGrid{};
  if (!g) return B200MDM_OK;
  if (!g->values) return fail(B200MDM_EINVAL, "%s: null values", what);
  if (g->gz < 2 || g->gx < 2 || static_cast<int64_t>(g->gz) * g->gx > (int64_t{1} << 30))
    return fail(B200MDM_EINVAL, "%s: %d x %d cells: at least 2 x 2, at most 2^30", what, g->gz, g->gx);
  if (!std::isfinite(g->cell) || g->cell <= 0.f) return fail(B200MDM_EINVAL, "%s: cell %g: a finite value > 0", what, g->cell);
  if (!std::isfinite(g->x0) || !std::isfinite(g->z0)) return fail(B200MDM_EINVAL, "%s: origin (%g, %g): finite values", what, g->x0, g->z0);
  const int64_t n = static_cast<int64_t>(g->gz) * g->gx;
  if (g->batch_stride != 0 && (g->batch_stride < n || g->batch_stride > (INT64_MAX - n) / std::max(B - 1, 1)))
    return fail(B200MDM_EINVAL, "%s: batch stride %lld: 0 (shared) or at least %lld, with %d samples", what,
                static_cast<long long>(g->batch_stride), static_cast<long long>(n), B);
  *out = SceneGrid{g->values, static_cast<long long>(g->batch_stride), g->gz, g->gx, g->x0, g->z0, g->cell};
  return B200MDM_OK;
}

// the scene terms over the foot terms `foot`, whose floor weight a terrain needs (nullptr: no foot terms to extend, which
// the setter refuses after these checks); floor_hint ends that message
static int fill_scene(float obstacle_weight, float obstacle_margin, const b200mdm_grid* sdf, const b200mdm_grid* terrain,
                      int B, const FootGuide* foot, const char* floor_hint, SceneGuide* out) {
  if (!std::isfinite(obstacle_weight) || obstacle_weight < 0.f || !std::isfinite(obstacle_margin) || obstacle_margin < 0.f)
    return fail(B200MDM_EINVAL, "obstacle weight %g, margin %g: finite values >= 0", obstacle_weight, obstacle_margin);
  TRY(check_grid(sdf, "obstacle sdf", B, &out->sdf));
  TRY(check_grid(terrain, "terrain", B, &out->terrain));
  if (obstacle_weight > 0.f && !sdf) return fail(B200MDM_EINVAL, "obstacle weight %g without an obstacle sdf", obstacle_weight);
  if (terrain && foot && foot->floor_w == 0.f) return fail(B200MDM_EINVAL, "a terrain needs a floor weight > 0%s", floor_hint);
  out->obstacle_w = obstacle_weight;
  out->margin = obstacle_margin;
  return B200MDM_OK;
}

// the interaction terms of motions of D features, with the reach rows in `rows` (the caller points out->pairs at them)
static int fill_inter(int32_t characters, float weight, float margin, const float* placement_dev, const int32_t* pairs_host,
                      int32_t n_pairs, const float* reach_host, const float* pair_weight_dev, int64_t pair_weight_stride, int B,
                      int T, int D, InterGuide* out, std::vector<InterPair>* rows) {
  if (characters < 2 || characters > IG_MAX_CHARS)
    return fail(B200MDM_EINVAL, "%d characters per scene: 2 .. %d", characters, IG_MAX_CHARS);
  if (B % characters) return fail(B200MDM_EINVAL, "batch %d is not a whole number of %d-character scenes", B, characters);
  if (!std::isfinite(weight) || weight < 0.f || !std::isfinite(margin) || margin < 0.f)
    return fail(B200MDM_EINVAL, "interaction weight %g, margin %g: finite values >= 0", weight, margin);
  if (!placement_dev) return fail(B200MDM_EINVAL, "null placement");
  if (n_pairs < 0 || n_pairs > B200MDM_MAX_INTERACTION_PAIRS)
    return fail(B200MDM_EINVAL, "%d reach rows: 0 .. %d", n_pairs, B200MDM_MAX_INTERACTION_PAIRS);
  if (n_pairs > 0 && (!pairs_host || !reach_host || !pair_weight_dev)) return fail(B200MDM_EINVAL, "null reach rows");
  if (n_pairs > 0 && pair_weight_stride != 0 && pair_weight_stride < static_cast<int64_t>(n_pairs) * T)
    return fail(B200MDM_EINVAL, "pair weight stride %lld: 0 (shared) or at least %lld", static_cast<long long>(pair_weight_stride),
                static_cast<long long>(n_pairs) * T);
  const int J = ric_dims(D).J;
  rows->resize(n_pairs);
  for (int n = 0; n < n_pairs; ++n) {
    const int32_t* r = pairs_host + 4 * n;
    if (r[0] < 0 || r[0] >= characters || r[2] < 0 || r[2] >= characters || r[0] == r[2] || r[1] < 0 || r[1] >= J ||
        r[3] < 0 || r[3] >= J)
      return fail(B200MDM_EINVAL, "reach row %d (%d, %d, %d, %d): characters in 0 .. %d and distinct, joints in 0 .. %d", n,
                  r[0], r[1], r[2], r[3], characters - 1, J - 1);
    if (!std::isfinite(reach_host[n]) || reach_host[n] < 0.f)
      return fail(B200MDM_EINVAL, "reach[%d] = %g: a finite value >= 0", n, reach_host[n]);
    (*rows)[n] = InterPair{r[0], r[1], r[2], r[3], reach_host[n]};
  }
  *out = InterGuide{placement_dev, nullptr, pair_weight_dev, static_cast<long long>(pair_weight_stride), characters, n_pairs,
                    weight, margin};
  return B200MDM_OK;
}

// ENOTIMPL unless a cluster of `characters` CTAs of `kern` (a kernel of the interaction terms' row) can be resident
template <class Kern>
static int check_inter_cluster(Kern kern, int characters, int B, int T, int D) {
  const size_t smem = GUIDE_VARIANTS[guide_variant(GT_INTER)].smem(T, ric_dims(D).R);
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(B);
  cfg.blockDim = dim3(JG_THREADS);
  cfg.dynamicSmemBytes = smem;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = static_cast<unsigned>(characters);
  at[0].val.clusterDim.y = 1;
  at[0].val.clusterDim.z = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  int n = 0;
  CUDA_TRY(cudaOccupancyMaxActiveClusters(&n, kern, &cfg));
  if (n < 1) return fail(B200MDM_ENOTIMPL, "a cluster of %d guidance CTAs (%zu B of shared memory each) cannot be resident",
                         characters, smem);
  return B200MDM_OK;
}

// The end of every guidance setter: h_guide goes up whole (it lives in the engine until the next call: no stream
// synchronisation), then `term` is on (0: the call turned its terms off)
static int upload_guide(b200mdm_engine* e, unsigned term, void* stream) {
  CUDA_TRY(cudaMemcpyAsync(e->jg_desc, &e->h_guide, sizeof(GuideDesc), cudaMemcpyHostToDevice,
                           static_cast<cudaStream_t>(stream)));
  e->guide_terms |= term;
  return B200MDM_OK;
}

extern "C" int b200mdm_set_joint_guidance(b200mdm_engine* e, const float* mean_dev, const float* std_dev,
                                          const float* target_dev, const float* weight_dev, float step, int32_t iters,
                                          void* stream) {
  if (!e) return fail(B200MDM_EINVAL, "null argument");
  JointGuide j;
  TRY(fill_joint(mean_dev, std_dev, target_dev, weight_dev, step, iters, &j));
  if (e->cfg.nfeats != 1 || (e->JF != 263 && e->JF != 251))
    return fail(B200MDM_EINVAL, "joint-position control needs the ric features of HumanML3D (263) or KIT (251) with nfeats 1 "
                "(got %d x %d)", e->cfg.njoints, e->cfg.nfeats);
  TRY(refuse(e, FAM_JOINT, F_PREFIX));
  if (!e->cond_set) return fail(B200MDM_ESTATE, "call b200mdm_set_cond / b200mdm_set_cond_dec first (they size the workspace)");
  TRY(refuse(e, FAM_JOINT));
  if (e->T > JG_MAX_FRAMES) return fail(B200MDM_ENOTIMPL, "joint-position control: at most %d frames", JG_MAX_FRAMES);
  if (!e->jg_desc) TRY(dalloc(&e->jg_desc, 1));
  if (!e->jg_x0) TRY(dalloc(&e->jg_x0, static_cast<size_t>(e->B) * e->JF * e->T));
  e->guide_terms = 0;
  e->h_guide = GuideDesc{};
  e->h_guide.j = j;
  return upload_guide(e, GT_JOINT, stream);
}

extern "C" int b200mdm_set_foot_guidance(b200mdm_engine* e, float contact_weight, float floor_weight, float floor_height,
                                         const float* contact_dev, const int64_t* lengths_host, void* stream) {
  if (!e) return fail(B200MDM_EINVAL, "null engine");
  FootGuide f;
  std::vector<int> len;
  TRY(fill_foot(contact_weight, floor_weight, floor_height, contact_dev, lengths_host, e->B, e->T, &f, &len));
  if (!(e->guide_terms & GT_JOINT)) return fail(B200MDM_ESTATE, "call b200mdm_set_joint_guidance first (foot guidance extends it)");
  e->guide_terms &= GT_FOOT - 1;
  if (lengths_host) {
    if (e->fg_len_cap < e->B) {
      dfree(e->fg_len);
      e->fg_len_cap = 0;
      TRY(dalloc(&e->fg_len, static_cast<size_t>(e->B)));
      e->fg_len_cap = e->B;
    }
    // the host staging lives in the engine until the next call: no stream synchronisation
    e->h_fg_len = std::move(len);
    CUDA_TRY(cudaMemcpyAsync(e->fg_len, e->h_fg_len.data(), e->B * sizeof(int), cudaMemcpyHostToDevice,
                             static_cast<cudaStream_t>(stream)));
    f.lengths = e->fg_len;
  }
  e->h_guide.f = f;
  e->h_guide.s = SceneGuide{};
  e->h_guide.i = InterGuide{};
  // both weights 0: plain joint-position control, with the lengths kept for the scene and interaction terms
  return upload_guide(e, contact_weight == 0.f && floor_weight == 0.f ? 0u : GT_FOOT, stream);
}

extern "C" int b200mdm_set_scene_guidance(b200mdm_engine* e, float obstacle_weight, float obstacle_margin,
                                          const b200mdm_grid* sdf, const b200mdm_grid* terrain, void* stream) {
  if (!e) return fail(B200MDM_EINVAL, "null engine");
  const bool joint = e->guide_terms & GT_JOINT;
  SceneGuide sg{};
  TRY(fill_scene(obstacle_weight, obstacle_margin, sdf, terrain, e->B, joint ? &e->h_guide.f : nullptr,
                 " (b200mdm_set_foot_guidance)", &sg));
  if (!joint) return fail(B200MDM_ESTATE, "call b200mdm_set_joint_guidance first (scene guidance extends it)");
  e->guide_terms &= GT_SCENE - 1;
  e->h_guide.s = sg;   // (kept when off: the interaction terms' scene)
  e->h_guide.i = InterGuide{};
  return upload_guide(e, obstacle_weight == 0.f && !terrain ? 0u : GT_SCENE, stream);   // off: no scene
}

extern "C" int b200mdm_set_interaction_guidance(b200mdm_engine* e, int32_t characters, float weight, float margin,
                                                const float* placement_dev, const int32_t* pairs_host, int32_t n_pairs,
                                                const float* reach_host, const float* pair_weight_dev,
                                                int64_t pair_weight_stride, void* stream) {
  if (!e) return fail(B200MDM_EINVAL, "null engine");
  if (!(e->guide_terms & GT_JOINT))
    return fail(B200MDM_ESTATE, "call b200mdm_set_joint_guidance first (interaction guidance extends it)");
  InterGuide ig;
  std::vector<InterPair> rows;
  TRY(fill_inter(characters, weight, margin, placement_dev, pairs_host, n_pairs, reach_host, pair_weight_dev,
                 pair_weight_stride, e->B, e->T, e->JF, &ig, &rows));
  TRY(init_kernel_attrs());
  TRY(check_inter_cluster(GUIDE_VARIANTS[guide_variant(GT_INTER)].step, characters, e->B, e->T, e->JF));
  e->guide_terms &= GT_INTER - 1;
  if (n_pairs > 0) {
    if (e->ig_pairs_cap < n_pairs) {
      dfree(e->ig_pairs);
      e->ig_pairs_cap = 0;
      TRY(dalloc(&e->ig_pairs, static_cast<size_t>(n_pairs)));
      e->ig_pairs_cap = n_pairs;
    }
    // the host staging lives in the engine until the next call: no stream synchronisation
    e->h_ig_pairs = std::move(rows);
    CUDA_TRY(cudaMemcpyAsync(e->ig_pairs, e->h_ig_pairs.data(), n_pairs * sizeof(InterPair), cudaMemcpyHostToDevice,
                             static_cast<cudaStream_t>(stream)));
  }
  ig.pairs = e->ig_pairs;
  e->h_guide.i = ig;
  return upload_guide(e, GT_INTER, stream);
}

extern "C" int b200mdm_set_prompt_weight(b200mdm_engine* e, int32_t K, const float* weight_dev, int64_t stride_b,
                                         int64_t stride_k, int64_t stride_f, int64_t stride_t, void* stream) {
  if (!e || !weight_dev) return fail(B200MDM_EINVAL, "null argument");
  if (stride_b < 0 || stride_k < 0 || stride_f < 0 || stride_t < 0) return fail(B200MDM_EINVAL, "negative weight stride");
  if (!e->cond_set || e->groups == 0)
    return fail(B200MDM_ESTATE, "call b200mdm_set_cond_multi / b200mdm_set_cond_multi_dec first (they clear the weights)");
  if (K != e->groups - 1) return fail(B200MDM_EINVAL, "%d prompt weights for %d prompts", K, e->groups - 1);
  if (!e->pw_desc) TRY(dalloc(&e->pw_desc, 1));
  e->h_pw = PromptWeight{weight_dev, stride_b, stride_k, stride_f, stride_t, K};
  CUDA_TRY(cudaMemcpyAsync(e->pw_desc, &e->h_pw, sizeof(PromptWeight), cudaMemcpyHostToDevice, static_cast<cudaStream_t>(stream)));
  e->pw_set = true;
  return B200MDM_OK;
}

// ------------------------------------------------------------------------------------------------ forward
struct StepArgs {
  int mode = B200MDM_MODE_X0;
  const float* x_in = nullptr;    // [B, JF, T] input to the denoiser (x_t)
  const float* noise = nullptr;   // explicit eps (single step); nullptr => tape from the device step state
  int const_noise = 0;
  int clip = 0;
  float* x_out = nullptr;
  float* pred = nullptr;
  bool explicit_t = false;        // use e->tvec instead of timestep_map[state.cur]
  bool philox = false;            // eps of this step is generated into e->eps_buf by the first kernel of the step
  int back = 0;                   // evaluate schedule index cur - back (PLMS improved Euler, second forward: 1)
  const float* x_step = nullptr;  // MODE_PLMS_EULER2: x_t of the step
  int order = 0;                  // MODE_PLMS_AB
  bool model_only = false;        // b200mdm_denoise: the bare model output, without the engine's inpainting
  bool slots = false;             // a schedule index per row (e->slots): OutStepSlots, philox_slots_kernel, slot_advance_kernel
};

// The per-step fields of the output step's parameters (p already holds the tables, the step state and the inpainting
// inputs): the output GEMM's epilogue and the joint-guidance step kernel read the same.
static void set_step_params(EpiOutParams* pp, const StepArgs& a, int B, int T, int JF) {
  EpiOutParams& p = *pp;
  p.x_t = a.x_in;
  p.noise = a.noise;
  p.x_out = a.x_out;
  p.pred_xstart = a.pred;
  p.x_step = a.x_step;
  p.noise_batch_stride = a.const_noise ? 0 : static_cast<long long>(JF) * T;
  p.B = B; p.T = T; p.J = JF; p.mode = a.mode;
  p.vb_chunks = (JF + 31) / 32;
  p.clip_denoised = a.clip;
  p.order = a.order;
  p.back = a.back;
}
// The output projection of the CFG-blended g16 rows with the update of a.mode fused into its epilogue, launched on the
// mode's GEMM instantiation.
static int launch_out_gemm(const CUtensorMap& m_g16, const CUtensorMap& m_wout, int B, int T, int JF, int d,
                           const StepArgs& a, EpiOutParams p, cudaStream_t s, int sms) {
  set_step_params(&p, a, B, T, JF);
  const int M = B * T, N = ((JF + 95) / 96) * 96, K = 3 * d;
  if (a.slots) return launch_gemm<96, EpiOut<OutStepSlots>>(m_g16, m_wout, M, N, K, p, s, sms);
  if (a.mode <= MODE_DDIM) return launch_gemm<96, EpiOut<OutStep>>(m_g16, m_wout, M, N, K, p, s, sms);
  if (a.mode == MODE_DDIM_REVERSE) return launch_gemm<96, EpiOut<OutReverse>>(m_g16, m_wout, M, N, K, p, s, sms);
  if (a.mode == MODE_DPM) return launch_gemm<96, EpiOut<OutDpm>>(m_g16, m_wout, M, N, K, p, s, sms);
  if (a.mode == MODE_VB) return launch_gemm<96, EpiOut<OutVb>>(m_g16, m_wout, M, N, K, p, s, sms);
  return launch_gemm<96, EpiOut<OutPlms>>(m_g16, m_wout, M, N, K, p, s, sms);
}

// Stage outputs requested by b200mdm_test_forward_taps: dst[id] (B200MDM_TAP_*) receives a device copy of the
// workspace buffer behind tap point id right after the launch that produces it; per-layer points only at `layer`.
struct ForwardTaps {
  int layer = 0;
  void* const* dst = nullptr;
  int n = 0;
  const int32_t* t_host = nullptr;   // the forward's timesteps: which temb_table rows B200MDM_TAP_TEMB gathers
};

// (source, bytes) of tap point id in the current workspace; bytes 0: the model kind has no such buffer.
static void tap_source(const b200mdm_engine* e, int id, const void** src, size_t* bytes) {
  const size_t M = e->M, d = e->d, h = sizeof(__half), f = sizeof(float), kw = e->kw, mem = static_cast<size_t>(e->Bp) * e->Mt;
  const bool dip = e->dec && !e->dec_clip;
  *src = nullptr;
  *bytes = 0;
  switch (id) {
    case B200MDM_TAP_EMBED: case B200MDM_TAP_TOK0: case B200MDM_TAP_L_IN: case B200MDM_TAP_L_LN1: case B200MDM_TAP_L_LN3:
      *src = e->hres; *bytes = M * 2 * d * h; break;
    case B200MDM_TAP_L_LN2:
      if (e->dec) { *src = e->hres; *bytes = M * 2 * d * h; }
      break;
    case B200MDM_TAP_CONDPROJ:
      if (!dip) { *src = e->condproj; *bytes = static_cast<size_t>(e->Bp) * d * f; }
      break;
    case B200MDM_TAP_TEMB: *src = e->temb_table; *bytes = static_cast<size_t>(e->B) * d * f; break;
    case B200MDM_TAP_MEM16: if (dip) { *src = e->mem16; *bytes = mem * 2 * d * h; } break;
    case B200MDM_TAP_KVC16: if (dip) { *src = e->kvc16; *bytes = mem * 2 * d * e->L * h; } break;
    case B200MDM_TAP_CROSS_C:
      if (e->dec_clip) { *src = e->cross_c; *bytes = static_cast<size_t>(e->L) * e->Bp * d * f; }
      break;
    case B200MDM_TAP_L_QKV: *src = e->qkv16; *bytes = M * 3 * d * h; break;
    case B200MDM_TAP_L_ATT: *src = e->att16; *bytes = M * kw * d * h; break;
    case B200MDM_TAP_L_QC: if (dip) { *src = e->qc16; *bytes = M * d * h; } break;
    case B200MDM_TAP_L_XATT: if (dip) { *src = e->att16; *bytes = M * kw * d * h; } break;
    case B200MDM_TAP_L_FFN: *src = e->ffn16; *bytes = M * kw * e->ff * h; break;
    case B200MDM_TAP_BLEND:
      *src = e->g16; *bytes = static_cast<size_t>(e->groups ? e->Bp : e->B) * e->T * 3 * d * h; break;
    case B200MDM_TAP_X0G:
      if (e->groups) { *src = e->mp_x0; *bytes = static_cast<size_t>(e->Bp) * e->JF * e->T * f; }
      break;
  }
}

extern "C" int64_t b200mdm_test_tap_bytes(const b200mdm_engine* e, int32_t id) {
  if (!e) return fail(B200MDM_EINVAL, "null engine");
  if (id < 0 || id >= B200MDM_TAP_COUNT) return fail(B200MDM_EINVAL, "tap point %d outside 0..%d", id, B200MDM_TAP_COUNT - 1);
  if (!e->cond_set) return fail(B200MDM_ESTATE, "no workspace: set the conditioning first");
  const void* src;
  size_t bytes;
  tap_source(e, id, &src, &bytes);
  return static_cast<int64_t>(bytes);
}

// Copy tap points first..last (layer l, or -1 outside the layer loop) into the caller's buffers, on stream s.
static int take_taps(const b200mdm_engine* e, const ForwardTaps& tp, int first, int last, int l, cudaStream_t s) {
  if (l >= 0 && l != tp.layer) return B200MDM_OK;
  for (int id = first; id <= last && id < tp.n; ++id) {
    if (!tp.dst[id]) continue;
    const void* src;
    size_t bytes;
    tap_source(e, id, &src, &bytes);
    if (bytes == 0) continue;   // (b200mdm_test_forward_taps rejects such requests up front)
    if (id == B200MDM_TAP_TEMB) {   // the rows temb_table[t_b] of this forward, b = 0..B-1
      const size_t row = static_cast<size_t>(e->d) * sizeof(float);
      for (int b = 0; b < e->B; ++b)
        CUDA_TRY(cudaMemcpyAsync(static_cast<char*>(tp.dst[id]) + b * row, e->temb_table + static_cast<size_t>(tp.t_host[b]) * e->d,
                                 row, cudaMemcpyDeviceToDevice, s));
      continue;
    }
    CUDA_TRY(cudaMemcpyAsync(tp.dst[id], src, bytes, cudaMemcpyDeviceToDevice, s));
  }
  return B200MDM_OK;
}

// The CLIP decoder's cross-attention rows of all layers at the step's timestep (tvec, or the step state's): out [L, Bp, d]
static int launch_cross_rows(const b200mdm_engine* e, float* out, const int* tvec, int back, cudaStream_t s) {
  CUDA_TRY(launch_k(cross_rows_kernel, dim3(e->Bp, e->L), dim3(128), 0, s, out, e->cross_b, e->cross_t, tvec, e->tmap, e->state,
                    e->B, e->Bp, e->d, e->cfg.temb_rows, back));
  return B200MDM_OK;
}

// Enqueue one denoiser forward (+ fused sampler step) on stream s.  Returns the number of kernels launched.
// taps: stage copies for b200mdm_test_forward_taps, nullptr everywhere else.
static int enqueue_forward(b200mdm_engine* e, const StepArgs& a, cudaStream_t s, int* n_kernels,
                           const ForwardTaps* taps = nullptr) {
  const int d = e->d, ff = e->ff, B = e->B, T = e->T, S = e->S, JF = e->JF, Kp = e->Kp_in;
  int nk = 0;
  PdlScope pdl_scope;
  if (a.philox && a.slots) {
    const long long n = static_cast<long long>(JF) * T;
    CUDA_TRY(launch_k(philox_slots_kernel, dim3(philox_blocks(B, n)), dim3(256), 0, s, e->eps_buf, B, n,
                      static_cast<const SlotState*>(e->slots)));
    ++nk;
  } else if (a.philox) {
    TRY(launch_philox(e->eps_buf, B, static_cast<long long>(JF) * T, 0ull, 0ll, 0u, e->state, s));
    ++nk;
  }
  if (a.mode == MODE_VB) {   // x_t = q_sample(x_start, i, eps): the denoiser's input
    TRY(launch_vb_xt(e->x_work, e->vb_xs, a.noise, e->tab[TAB_VB], e->state, static_cast<size_t>(B) * JF * T, s));
    ++nk;
  }
  TRY(launch_pack_input(a.x_in, e->xin16, B, JF, T, S, Kp, e->s_off, s));
  TRY(launch_embed_gemm(e->m_xin, e->m_win, e->m_res_c, e->m_res_u, e->pe_bias, e->MB, S, d, Kp, e->halves > 1 || e->groups > 1 ? 2 : 1,
                        s, e->num_sms));
  nk += 2;
  // multi-prompt guidance: the first and last groups came from the launch above, the groups between them in pairs
  for (int g = 1; g < e->groups - 1; g += 2) {
    const int pair = g + 1 < e->groups - 1 ? 2 : 1;
    CUtensorMap m_a, m_b;
    TRY(make_map_res(&m_a, e->hres + static_cast<size_t>(g) * e->MB * d * 2, e->MB, d));
    TRY(make_map_res(&m_b, e->hres + static_cast<size_t>(g + pair - 1) * e->MB * d * 2, e->MB, d));
    TRY(launch_embed_gemm(e->m_xin, e->m_win, m_a, m_b, e->pe_bias, e->MB, S, d, Kp, pair, s, e->num_sms));
    ++nk;
  }
  if (taps) TRY(take_taps(e, *taps, B200MDM_TAP_EMBED, B200MDM_TAP_EMBED, -1, s));
  const float* target_g = e->target_set ? e->tgt_g : nullptr;   // timestep embedding + target (model/mdm.py:197-199)
  if (!e->dec || e->dec_clip) {
    // token 0: cond + (temb + g) (encoder), or the decoder's timestep token (temb + g) without the text (mdm.py:256)
    CUDA_TRY(launch_k(tok0_rows_kernel, dim3(e->Bp), dim3(128), 0, s, e->hres, e->dec_clip ? nullptr : e->condproj,
                      e->temb_table, e->pe, a.explicit_t ? e->tvec : nullptr, e->tmap, e->state, target_g, B, S, d,
                      e->cfg.temb_rows, a.back));
    if (e->dec_clip) {
      // every layer's cross-attention row of this step: c_l[b'] = cb_l[b'] + ct_l[t]
      TRY(launch_cross_rows(e, e->cross_c, a.explicit_t ? e->tvec : nullptr, a.back, s));
      ++nk;
    }
  } else {
    // cross-attention memory of this step: text tokens + timestep embedding (model/mdm.py:218-220)
    CUDA_TRY(launch_k(mem_build_kernel, dim3(e->Mt, e->Bp), dim3(128), 0, s, e->mem16, e->memproj, e->temb_table,
                      a.explicit_t ? e->tvec : nullptr, e->tmap, e->state, target_g, B, e->Mt, d, e->cfg.temb_rows, a.back));
    // ... and its key / value projections for every layer in one GEMM (N = L * 2d; hi half of the memory, K = d)
    EpiBiasF16Global::Params p{e->bkv_all};
    TRY((launch_gemm_pp<EpiBiasF16Global>(e->m_mem, e->m_wkv_all, e->m_kvc_st, e->Bp * e->Mt, e->L * 2 * d, d, p, s, e->num_sms)));
    ++nk;
  }
  ++nk;
  if (taps) TRY(take_taps(e, *taps, B200MDM_TAP_TOK0, B200MDM_TAP_KVC16, -1, s));
  const int kw = e->kw;
  const bool wide = kw == 2;
  for (int l = 0; l < e->L; ++l) {
    const LayerW& w = e->layers[l];
    if (taps) TRY(take_taps(e, *taps, B200MDM_TAP_L_IN, B200MDM_TAP_L_IN, l, s));
    if (B200_SKIP(1)) {
      ++nk;
    } else {
      {
        // trans_dec keeps [hi | lo] activations only where the precision study needs them (self-attention output,
        // FFN-up input, FFN-down input: oracle emulation 6.2e-4 vs 5.1e-4 with every site split, tolerance 1e-3); the
        // projections below read the hi half alone: K = d against the first d columns of [W | W]
        TRY((launch_gemm_bias<false>(e->m_h16, w.m_wqkv, e->m_qkv_st, e->M, 3 * d, d, w.bqkv, s, e->num_sms)));
      }
      if (taps) TRY(take_taps(e, *taps, B200MDM_TAP_L_QKV, B200MDM_TAP_L_QKV, l, s));
      TRY(launch_attention_tc(e->m_qkv_kv, e->qkv16, e->att16, e->kvlen, e->Bp, S, d, e->H, s, wide));
      if (taps) TRY(take_taps(e, *taps, B200MDM_TAP_L_ATT, B200MDM_TAP_L_ATT, l, s));
    }
    if (!B200_SKIP(2)) TRY(launch_gemm_resid_ln(e->m_att, w.m_wo_256, e->m_hres, e->M, kw * d, w.bo, w.g1, w.be1, s, e->num_sms));
    if (taps) TRY(take_taps(e, *taps, B200MDM_TAP_L_LN1, B200MDM_TAP_L_LN1, l, s));
    if (e->dec_clip) {
      // cross-attention block over the one-token memory + norm2: h <- LN2(h + c_l[b'])
      TRY(launch_row_bias_ln(e->hres, e->cross_c + static_cast<size_t>(l) * e->Bp * d, w.g2, w.be2, e->M, S, s));
      ++nk;
    } else if (e->dec) {
      // cross-attention block of nn.TransformerDecoderLayer: q from the sequence, k/v from the text memory
      TRY((launch_gemm_bias<false>(e->m_h16, w.m_wq_c, e->m_qc_st, e->M, d, d, w.bq_c, s, e->num_sms)));
      if (taps) TRY(take_taps(e, *taps, B200MDM_TAP_L_QC, B200MDM_TAP_L_QC, l, s));
      // kv: this layer's k | v columns of the all-layer memory projection
      TRY(launch_cross_attention(e->qc16, e->kvc16 + static_cast<size_t>(l) * 2 * d, e->memmask, e->att16, e->Bp, S, e->Mt, d,
                                 e->H, e->L * 2 * d, s));
      if (taps) TRY(take_taps(e, *taps, B200MDM_TAP_L_XATT, B200MDM_TAP_L_XATT, l, s));
      TRY(launch_gemm_resid_ln(e->m_att, w.m_wo_c_256, e->m_hres, e->M, d, w.bo_c, w.g2, w.be2, s, e->num_sms));   // cross-attention output: hi half
      nk += 3;
    }
    if (taps) TRY(take_taps(e, *taps, B200MDM_TAP_L_LN2, B200MDM_TAP_L_LN2, l, s));
    if (wide) {
      EpiBiasF16Wide<true>::Params p{w.b1, ff};
      TRY((launch_gemm_pp<EpiBiasF16Wide<true>>(e->m_h16, w.m_w1, e->m_ffn_st, e->M, ff, kw * d, p, s, e->num_sms)));
    } else if (!B200_SKIP(4)) {
      TRY((launch_gemm_bias<true>(e->m_h16, w.m_w1, e->m_ffn_st, e->M, ff, d, w.b1, s, e->num_sms)));
    }
    if (taps) TRY(take_taps(e, *taps, B200MDM_TAP_L_FFN, B200MDM_TAP_L_FFN, l, s));
    if (!B200_SKIP(8)) TRY(launch_gemm_resid_ln(e->m_ffn, w.m_w2_256, e->m_hres, e->M, kw * ff, w.b2, e->dec ? w.g3 : w.g2,
                             e->dec ? w.be3 : w.be2, s, e->num_sms));
    if (taps) TRY(take_taps(e, *taps, B200MDM_TAP_L_LN3, B200MDM_TAP_L_LN3, l, s));
    nk += 5;
  }
  // multi-prompt guidance: every group's frame rows are split as they are (halves 1 over G * B motions)
  const int G = e->groups, GB = G ? G * B : B;
  TRY(launch_blend_split(e->hres, e->g16, e->scale, GB, S, T, e->s_off, d, G ? 1 : e->halves, e->hs_set ? e->hs_desc : nullptr, s));
  ++nk;
  if (taps) TRY(take_taps(e, *taps, B200MDM_TAP_BLEND, B200MDM_TAP_BLEND, -1, s));
  {
    EpiOutParams p{};
    p.bias = e->b_out;
    // inpainting belongs to the sampler (p_mean_variance, gaussian_diffusion.py:300-304), not to MDM.forward
    p.inpaint_mask = a.model_only ? nullptr : e->inpaint_mask;
    p.inpaint_weight = a.model_only ? nullptr : e->inpaint_weight;
    p.inpaint_motion = a.model_only ? nullptr : e->inpaint_motion;
    set_tables(&p, e->tab);
    p.eps_ring = e->plms_ring;
    p.x0_hist = e->dpm_hist;
    p.x_start = e->vb_xs;
    p.vb_part = e->vb_part;
    p.state = e->state;
    p.slots = e->slots;
    if (G) {
      // multi-prompt guidance: the output GEMM writes every group's raw x0, compose_step_kernel composes it and runs the
      // step's tail (the bare model output too: b200mdm_denoise composes, without inpainting)
      StepArgs ax = a;
      ax.mode = MODE_X0;
      ax.x_out = e->mp_x0;
      ax.pred = nullptr;
      ax.clip = 0;
      EpiOutParams px = p;
      px.inpaint_mask = nullptr;
      px.inpaint_weight = nullptr;
      px.inpaint_motion = nullptr;
      TRY(launch_out_gemm(e->m_g16, e->m_wout, GB, T, JF, d, ax, px, s, e->num_sms));
      if (taps) TRY(take_taps(e, *taps, B200MDM_TAP_X0G, B200MDM_TAP_X0G, -1, s));
      set_step_params(&p, a, B, T, JF);
      const dim3 grid(static_cast<unsigned>((static_cast<size_t>(JF) * T + MP_THREADS - 1) / MP_THREADS), B);
      const PromptWeight* pw = e->pw_desc;
      const float* x0g = e->mp_x0;
      if (a.mode <= MODE_DDIM) CUDA_TRY(launch_k(compose_step_kernel<OutStep>, grid, dim3(MP_THREADS), 0, s, pw, x0g, p));
      else if (a.mode == MODE_DDIM_REVERSE) CUDA_TRY(launch_k(compose_step_kernel<OutReverse>, grid, dim3(MP_THREADS), 0, s, pw, x0g, p));
      else if (a.mode == MODE_DPM) CUDA_TRY(launch_k(compose_step_kernel<OutDpm>, grid, dim3(MP_THREADS), 0, s, pw, x0g, p));
      else   // PLMS: the variational bound refuses multi-prompt guidance (REFUSED)
        CUDA_TRY(launch_k(compose_step_kernel<OutPlms>, grid, dim3(MP_THREADS), 0, s, pw, x0g, p));
      nk += 2;
    } else if (e->guide_terms && !a.model_only) {
      // joint-position control: the output GEMM writes the raw x0, the guidance kernel runs the step's tail on it
      StepArgs ax = a;
      ax.mode = MODE_X0;
      ax.x_out = e->jg_x0;
      ax.pred = nullptr;
      ax.clip = 0;
      EpiOutParams px = p;
      px.inpaint_mask = nullptr;
      px.inpaint_weight = nullptr;
      px.inpaint_motion = nullptr;
      TRY(launch_out_gemm(e->m_g16, e->m_wout, B, T, JF, d, ax, px, s, e->num_sms));
      set_step_params(&p, a, B, T, JF);
      const GuideVariant& v = GUIDE_VARIANTS[guide_variant(e->guide_terms)];
      CUDA_TRY(launch_kc(v.step, dim3(B), dim3(JG_THREADS), v.smem(T, ric_dims(JF).R), s, v.clusters ? e->h_guide.i.chars : 0,
                         static_cast<const GuideDesc*>(e->jg_desc), static_cast<const float*>(e->jg_x0), p));
      nk += 2;
    } else {
      TRY(launch_out_gemm(e->m_g16, e->m_wout, B, T, JF, d, a, p, s, e->num_sms));
      ++nk;
    }
  }
  if (a.mode == MODE_VB) {
    TRY(launch_vb_reduce(e->vb_terms, e->vb_cap, e->vb_part, B, T, JF, e->state, s));
    ++nk;
  }
  *n_kernels = nk;
  return B200MDM_OK;
}

static int check_ready(b200mdm_engine* e, bool need_sched) {
  if (!e) return fail(B200MDM_EINVAL, "null engine");
  if (!e->finalized) return fail(B200MDM_ESTATE, "weights not finalised");
  if (!e->cond_set) return fail(B200MDM_ESTATE, "b200mdm_set_cond has not been called");
  if (e->dec && e->ctx > 0 && !e->prefix_set) return fail(B200MDM_ESTATE, "b200mdm_set_prefix has not been called (y['prefix'])");
  if (need_sched && e->n_steps <= 0) return fail(B200MDM_ESTATE, "b200mdm_set_schedule has not been called");
  if (e->groups && !e->pw_set) return fail(B200MDM_ESTATE, "b200mdm_set_prompt_weight has not been called");
  return B200MDM_OK;
}

// EINVAL unless flags holds nothing outside `allowed`: B200MDM_FLAG_CLIP_DENOISED, with or without
// B200MDM_FLAG_PHILOX_NOISE.
static int check_flags(const char* family, int32_t flags, int32_t allowed) {
  if (!(flags & ~allowed)) return B200MDM_OK;
  return fail(B200MDM_EINVAL, "%s takes no flag but B200MDM_FLAG_CLIP_DENOISED%s", family,
              (allowed & B200MDM_FLAG_PHILOX_NOISE) ? " and B200MDM_FLAG_PHILOX_NOISE" : "");
}

static int check_timesteps(const b200mdm_engine* e, const int32_t* timesteps_host) {
  for (int b = 0; b < e->B; ++b)
    if (timesteps_host[b] < 0 || timesteps_host[b] >= e->cfg.temb_rows)
      return fail(B200MDM_EINVAL, "timestep %d outside the pre-embedded range [0, %d)", timesteps_host[b], e->cfg.temb_rows);
  return B200MDM_OK;
}

// One model forward at explicit per-sample timesteps (b200mdm_denoise; with taps, b200mdm_test_forward_taps).
static int denoise_forward(b200mdm_engine* e, const float* x_dev, const int32_t* timesteps_host, float* out_dev,
                           cudaStream_t s, const ForwardTaps* taps, int* n_kernels) {
  CUDA_TRY(cudaMemcpyAsync(e->tvec, timesteps_host, e->B * sizeof(int), cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaStreamSynchronize(s));  // timesteps_host is caller memory
  StepArgs a;
  a.mode = B200MDM_MODE_X0;
  a.x_in = x_dev;
  a.x_out = out_dev;
  a.explicit_t = true;
  a.model_only = true;
  return enqueue_forward(e, a, s, n_kernels, taps);
}

extern "C" int b200mdm_denoise(b200mdm_engine* e, const float* x_dev, const int32_t* timesteps_host, float* out_dev,
                               void* stream) {
  TRY(check_ready(e, false));
  if (!x_dev || !timesteps_host || !out_dev) return fail(B200MDM_EINVAL, "null tensor");
  TRY(check_timesteps(e, timesteps_host));
  int nk = 0;
  TRY(denoise_forward(e, x_dev, timesteps_host, out_dev, static_cast<cudaStream_t>(stream), nullptr, &nk));
  e->launches += nk;
  return B200MDM_OK;
}

extern "C" int b200mdm_test_forward_taps(b200mdm_engine* e, const float* x_dev, const int32_t* timesteps_host, float* out_dev,
                                         int32_t layer, void* const* tap_dev, int32_t n_taps, void* stream) {
  if (!e || !x_dev || !timesteps_host || !out_dev) return fail(B200MDM_EINVAL, "null argument");
  if (n_taps < 0 || n_taps > B200MDM_TAP_COUNT || (n_taps > 0 && !tap_dev))
    return fail(B200MDM_EINVAL, "n_taps %d: 0..%d tap buffers (tap_dev may be NULL only with n_taps 0)", n_taps, B200MDM_TAP_COUNT);
  TRY(check_ready(e, false));
  if (layer < 0 || layer >= e->L) return fail(B200MDM_EINVAL, "layer %d outside [0, %d)", layer, e->L);
  TRY(check_timesteps(e, timesteps_host));
  for (int id = 0; id < n_taps; ++id) {
    const void* src;
    size_t bytes;
    tap_source(e, id, &src, &bytes);
    if (tap_dev[id] && bytes == 0) return fail(B200MDM_EINVAL, "tap point %d does not exist in this model", id);
  }
  ForwardTaps tp;
  tp.layer = layer;
  tp.dst = tap_dev;
  tp.n = n_taps;
  tp.t_host = timesteps_host;
  int nk = 0;
  return denoise_forward(e, x_dev, timesteps_host, out_dev, static_cast<cudaStream_t>(stream), &tp, &nk);
}

extern "C" int b200mdm_sample_step(b200mdm_engine* e, int32_t mode, int32_t index, const float* x_t_dev,
                                   const float* noise_dev, int32_t flags, float* x_out_dev,
                                   float* pred_xstart_dev, void* stream) {
  TRY(check_ready(e, true));
  const bool reverse = mode == B200MDM_MODE_DDIM_REVERSE;
  if (mode != B200MDM_MODE_DDPM && mode != B200MDM_MODE_DDIM && !reverse) return fail(B200MDM_EINVAL, "bad mode");
  if (index < 0 || index >= e->n_steps) return fail(B200MDM_EINVAL, "schedule index out of range");
  if (!x_t_dev || (!noise_dev && !reverse) || !x_out_dev) return fail(B200MDM_EINVAL, "null tensor");
  if (reverse) {
    TRY(check_flags("DDIM inversion", flags, B200MDM_FLAG_CLIP_DENOISED));
    TRY(need_table(e, TAB_NEXT));
    TRY(refuse(e, FAM_REVERSE));
  }
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  step_set_kernel<<<1, 1, 0, s>>>(e->state, 0, index, nullptr, 0, e->noise_seed, e->noise_sample_base, e->n_steps);
  CUDA_TRY(cudaGetLastError());
  StepArgs a;
  a.mode = mode;
  a.x_in = x_t_dev;
  a.noise = noise_dev;
  a.const_noise = flags & B200MDM_FLAG_CONST_NOISE;
  a.clip = (flags & B200MDM_FLAG_CLIP_DENOISED) ? 1 : 0;
  a.x_out = x_out_dev;
  a.pred = pred_xstart_dev;
  int nk = 0;
  TRY(enqueue_forward(e, a, s, &nk));
  e->launches += nk + 1;
  return B200MDM_OK;
}

// Move the step state to the next step of the loop: down the schedule, or up it for the DDIM inversion.
static cudaError_t launch_advance(b200mdm_engine* e, const StepArgs& a, cudaStream_t s) {
  PdlScope pdl_scope;
  if (a.slots)
    return launch_k(slot_advance_kernel, dim3((e->B + 127) / 128), dim3(128), 0, s, e->slots, e->tvec,
                    static_cast<const int*>(e->tmap), e->B);
  return launch_k(step_advance_kernel, dim3(1), dim3(1), 0, s, e->state, a.mode == MODE_DDIM_REVERSE ? 1 : -1);
}

// Make the workspace's step graph (one forward + step_advance, captured on the engine stream) the graph of `key`.
static int ensure_step_graph(b200mdm_engine* e, const GraphKey& key, const StepArgs& a) {
  if (e->graph_exec && key == e->graph_key) return B200MDM_OK;
  drop_graph(e);
  cudaGraph_t graph = nullptr;
  CUDA_TRY(cudaStreamBeginCapture(e->work, cudaStreamCaptureModeThreadLocal));
  int nk = 0;
  int r = enqueue_forward(e, a, e->work, &nk);
  if (r == B200MDM_OK && launch_advance(e, a, e->work) != cudaSuccess)
    r = fail(B200MDM_ECUDA, "step_advance launch failed during capture");
  cudaError_t ce = cudaStreamEndCapture(e->work, &graph);
  if (r != B200MDM_OK) {
    if (graph) cudaGraphDestroy(graph);
    return r;
  }
  if (ce != cudaSuccess) return fail(B200MDM_ECUDA, "graph capture failed: %s", cudaGetErrorString(ce));
  ce = cudaGraphInstantiate(&e->graph_exec, graph, 0);
  cudaGraphDestroy(graph);
  if (ce != cudaSuccess) {
    e->graph_exec = nullptr;
    return fail(B200MDM_ECUDA, "graph instantiate failed: %s", cudaGetErrorString(ce));
  }
  e->graph_key = key;
  e->graph_kernels = nk + 1;
  return B200MDM_OK;
}

// One step of a loop on s: a replay of the step graph, or the same forward + step_advance as plain launches.
static int enqueue_step(b200mdm_engine* e, const StepArgs& a, cudaStream_t s, bool use_graph) {
  if (use_graph) {
    CUDA_TRY(cudaGraphLaunch(e->graph_exec, s));
    e->launches += e->graph_kernels;
    return B200MDM_OK;
  }
  int nk = 0;
  TRY(enqueue_forward(e, a, s, &nk));
  CUDA_TRY(launch_advance(e, a, s));
  e->launches += nk + 1;
  return B200MDM_OK;
}

// The pseudo improved-Euler step (gaussian_diffusion.py:1042-1049) at the schedule index the step state holds:
// forward 1 at (x_t, i) leaves eps0 in the ring, x0 in plms_pred and mean1 in plms_mid; forward 2 at (mean1, i - 1)
// writes the sample to x_out.  Then the step state advances.
static int enqueue_plms_euler(b200mdm_engine* e, const StepArgs& base, const float* x_t, float* x_out, cudaStream_t s) {
  StepArgs a = base;
  a.mode = MODE_PLMS_EULER1;
  a.x_in = x_t;
  a.x_out = e->plms_mid;
  a.pred = e->plms_pred;
  int nk1 = 0, nk2 = 0;
  TRY(enqueue_forward(e, a, s, &nk1));
  a.mode = MODE_PLMS_EULER2;
  a.x_in = e->plms_mid;
  a.x_step = x_t;
  a.x_out = x_out;
  a.back = 1;
  TRY(enqueue_forward(e, a, s, &nk2));
  CUDA_TRY(launch_advance(e, a, s));
  e->launches += nk1 + nk2 + 1;
  return B200MDM_OK;
}

// n_run steps of `a` from schedule index first_index on the engine's working buffer (a.x_in == a.x_out == x_work), with
// the step counter starting at `done`; plms_euler: the first step is the PLMS improved-Euler step (two forwards, never
// a graph), the rest are steps of `a`.  x_in_dev == NULL continues from the state the previous call left there;
// x_out_dev == NULL leaves the result there.
// The stream a loop of `a` runs on: the graph path runs on the engine's own stream (the caller's may be the legacy
// default stream, which cannot be captured), ordered after the caller's stream with an event (loop_leave orders it
// back).  x_work no longer holds a PLMS, DPM-Solver++ or chain loop to continue.
static int loop_enter(b200mdm_engine* e, const StepArgs& a, int32_t flags, int32_t use_graph, cudaStream_t user,
                      cudaStream_t* s) {
  *s = use_graph ? e->work : user;
  if (!use_graph) attach_l2_window(e, user);   // plain launches: the residual-stream window goes on the caller's stream
  if (use_graph) {
    GraphKey key;
    key.mode = a.mode; key.B = e->B; key.T = e->T; key.flags = flags; key.order = a.order;
    key.imask = e->inpaint_mask; key.iweight = e->inpaint_weight; key.imotion = e->inpaint_motion;
    key.target_g = e->target_set ? e->tgt_g : nullptr;
    key.hs = e->hs_set ? e->hs_desc : nullptr;
    key.guide = guide_variant(e->guide_terms);
    key.chars = key.guide >= 0 && GUIDE_VARIANTS[key.guide].clusters ? e->h_guide.i.chars : 0;
    key.groups = e->groups;
    key.slots = a.slots;
    TRY(ensure_step_graph(e, key, a));
    CUDA_TRY(cudaEventRecord(e->ev_in, user));
    CUDA_TRY(cudaStreamWaitEvent(e->work, e->ev_in, 0));
  }
  e->plms_done = -1;
  e->dpm_done = -1;
  e->chain_next = -1;
  return B200MDM_OK;
}

static int loop_leave(b200mdm_engine* e, int32_t use_graph, cudaStream_t user) {
  if (use_graph) {
    CUDA_TRY(cudaEventRecord(e->ev_out, e->work));
    CUDA_TRY(cudaStreamWaitEvent(user, e->ev_out, 0));
  }
  return B200MDM_OK;
}

static int run_loop(b200mdm_engine* e, const StepArgs& a, int32_t flags, int32_t first_index, int32_t n_run,
                    const float* x_in_dev, float* x_out_dev, const float* noise_tape_dev, int64_t noise_step_stride,
                    int32_t use_graph, void* stream, int done = 0, bool plms_euler = false) {
  cudaStream_t user = static_cast<cudaStream_t>(stream);
  const size_t x_bytes = static_cast<size_t>(e->B) * e->JF * e->T * sizeof(float);
  cudaStream_t s;
  TRY(loop_enter(e, a, flags, use_graph, user, &s));
  if (x_in_dev) CUDA_TRY(cudaMemcpyAsync(e->x_work, x_in_dev, x_bytes, cudaMemcpyDeviceToDevice, s));
  step_set_kernel<<<1, 1, 0, s>>>(e->state, done, first_index, noise_tape_dev, noise_step_stride, e->noise_seed,
                                  e->noise_sample_base, e->n_steps);
  CUDA_TRY(cudaGetLastError());
  e->launches += 1;
  int k = 0;
  if (plms_euler) {
    TRY(enqueue_plms_euler(e, a, e->x_work, e->x_work, s));
    k = 1;
  }
  for (; k < n_run; ++k) TRY(enqueue_step(e, a, s, use_graph));
  if (a.mode == MODE_PLMS_AB) {
    e->plms_done = done + n_run;
    e->plms_order = a.order;
  } else if (a.mode == MODE_DPM) {
    e->dpm_done = done + n_run;
    e->dpm_order = a.order;
  }
  if (x_out_dev) CUDA_TRY(cudaMemcpyAsync(x_out_dev, e->x_work, x_bytes, cudaMemcpyDeviceToDevice, s));
  return loop_leave(e, use_graph, user);
}

// EINVAL unless schedule indices first_index, first_index - 1, ... (n_run of them) exist.
static int check_range_down(const b200mdm_engine* e, int32_t first_index, int32_t n_run) {
  if (n_run <= 0 || first_index >= e->n_steps || first_index - n_run + 1 < 0) return fail(B200MDM_EINVAL, "bad step range");
  return B200MDM_OK;
}

// The StepArgs of a loop of `mode`.  The loop runs in place on an engine-owned buffer (fixed address => the captured
// step graph never changes); every element is read and written by the same thread of the fused output epilogue.
static StepArgs loop_args(b200mdm_engine* e, int mode, int order, int32_t flags, bool philox) {
  StepArgs a;
  a.mode = mode;
  a.order = order;
  a.x_in = e->x_work;
  a.x_out = e->x_work;
  a.noise = philox ? e->eps_buf : nullptr;
  a.philox = philox;
  a.const_noise = flags & B200MDM_FLAG_CONST_NOISE;
  a.clip = (flags & B200MDM_FLAG_CLIP_DENOISED) ? 1 : 0;
  return a;
}

// A loop's device buffers, all or nothing: each null pointer gets its n floats; after a failure every one of them is
// freed, so that no later call finds a partial set.
struct LoopBuf {
  float** p;
  size_t n;
};
static int alloc_all(std::initializer_list<LoopBuf> bufs) {
  int r = B200MDM_OK;
  for (const LoopBuf& b : bufs)
    if (r == B200MDM_OK && !*b.p) r = dalloc(b.p, b.n);
  if (r != B200MDM_OK)
    for (const LoopBuf& b : bufs) dfree(*b.p);
  return r;
}

// Schedule indices first_index, first_index-1, ... (n_run of them) on the engine's working buffer.
extern "C" int b200mdm_sample_loop_range(b200mdm_engine* e, int32_t mode, int32_t first_index, int32_t n_run,
                                         const float* x_in_dev, float* x_out_dev, const float* noise_tape_dev,
                                         int64_t noise_step_stride, int32_t flags, int32_t use_graph, void* stream) {
  TRY(check_ready(e, true));
  if (mode != B200MDM_MODE_DDPM && mode != B200MDM_MODE_DDIM) return fail(B200MDM_EINVAL, "bad mode");
  TRY(check_range_down(e, first_index, n_run));
  const bool philox = (flags & B200MDM_FLAG_PHILOX_NOISE) != 0;
  if (!philox && !noise_tape_dev) return fail(B200MDM_EINVAL, "null noise tape (or pass B200MDM_FLAG_PHILOX_NOISE)");
  return run_loop(e, loop_args(e, mode, 0, flags, philox), flags, first_index, n_run, x_in_dev, x_out_dev, noise_tape_dev,
                  noise_step_stride, use_graph, stream);
}

extern "C" int b200mdm_sample_loop(b200mdm_engine* e, int32_t mode, int32_t skip_timesteps, const float* x_T_dev,
                                   float* x_0_dev, const float* noise_tape_dev, int64_t noise_step_stride,
                                   int32_t flags, int32_t use_graph, void* stream) {
  TRY(check_ready(e, true));
  if (skip_timesteps < 0 || skip_timesteps >= e->n_steps) return fail(B200MDM_EINVAL, "bad skip_timesteps");
  if (!x_T_dev || !x_0_dev) return fail(B200MDM_EINVAL, "null tensor");
  return b200mdm_sample_loop_range(e, mode, e->n_steps - 1 - skip_timesteps, e->n_steps - skip_timesteps, x_T_dev, x_0_dev,
                                   noise_tape_dev, noise_step_stride, flags, use_graph, stream);
}

// ------------------------------------------------------------------------------------------------ continuous batching
// DESIGN.md, "Continuous batching".  Every row of the workspace is a slot running its own request at its own schedule
// index; the step graph is the uniform one with three kernels swapped for their slot variants (philox_slots_kernel,
// EpiOut<OutStepSlots>, slot_advance_kernel), and the forward reads the per-row timesteps through its explicit_t path.
static int ensure_slots(b200mdm_engine* e) {
  if (!e->slots) TRY(dalloc(&e->slots, e->B));
  return B200MDM_OK;
}

extern "C" int b200mdm_sample_step_at(b200mdm_engine* e, int32_t mode, const int32_t* index_host, const float* x_t_dev,
                                      const float* noise_dev, int32_t flags, float* x_out_dev, float* pred_xstart_dev,
                                      void* stream) {
  TRY(check_ready(e, true));
  if (mode != B200MDM_MODE_DDPM && mode != B200MDM_MODE_DDIM) return fail(B200MDM_EINVAL, "bad mode");
  if (!index_host || !x_t_dev || !noise_dev || !x_out_dev) return fail(B200MDM_EINVAL, "null argument");
  if (flags & B200MDM_FLAG_CONST_NOISE)
    return fail(B200MDM_ENOTIMPL, "B200MDM_FLAG_CONST_NOISE with a schedule index per sample is not implemented");
  TRY(check_flags("b200mdm_sample_step_at", flags, B200MDM_FLAG_CLIP_DENOISED));
  for (int b = 0; b < e->B; ++b)
    if (index_host[b] < 0 || index_host[b] >= e->n_steps) return fail(B200MDM_EINVAL, "schedule index out of range");
  TRY(refuse(e, FAM_STEP_AT));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  TRY(ensure_slots(e));
  e->slot_mode = false;   // the step overwrites the slot state
  e->h_slot_idx.assign(index_host, index_host + e->B);
  CUDA_TRY(cudaMemcpyAsync(e->tvec, e->h_slot_idx.data(), e->B * sizeof(int), cudaMemcpyHostToDevice, s));
  slots_from_index_kernel<<<(e->B + 127) / 128, 128, 0, s>>>(e->slots, e->tvec, e->tmap, e->B);
  CUDA_TRY(cudaGetLastError());
  StepArgs a;
  a.mode = mode;
  a.x_in = x_t_dev;
  a.noise = noise_dev;
  a.clip = (flags & B200MDM_FLAG_CLIP_DENOISED) ? 1 : 0;
  a.x_out = x_out_dev;
  a.pred = pred_xstart_dev;
  a.explicit_t = true;
  a.slots = true;
  int nk = 0;
  TRY(enqueue_forward(e, a, s, &nk));
  e->launches += nk + 1;
  return B200MDM_OK;
}

extern "C" int b200mdm_slots_begin(b200mdm_engine* e, int32_t slots, int32_t nframes, int32_t guided, int32_t mode,
                                   int32_t flags, void* stream) {
  if (!e) return fail(B200MDM_EINVAL, "null engine");
  if (!e->finalized) return fail(B200MDM_ESTATE, "weights not finalised");
  if (e->n_steps <= 0) return fail(B200MDM_ESTATE, "b200mdm_set_schedule has not been called");
  if (slots <= 0 || nframes <= 0) return fail(B200MDM_EINVAL, "bad slots / nframes");
  if (mode != B200MDM_MODE_DDPM && mode != B200MDM_MODE_DDIM)
    return fail(B200MDM_ENOTIMPL, "continuous batching runs DDPM and DDIM (PLMS, DPM-Solver++, DDIM inversion and the "
                "bound carry history or tables that are not per slot)");
  if (flags & B200MDM_FLAG_CONST_NOISE) return fail(B200MDM_ENOTIMPL, "B200MDM_FLAG_CONST_NOISE with continuous batching");
  TRY(check_flags("continuous batching", flags, B200MDM_FLAG_CLIP_DENOISED | B200MDM_FLAG_PHILOX_NOISE));
  if (e->dec && !e->dec_clip) return fail(B200MDM_ENOTIMPL, "continuous batching with BERT text memories is not implemented");
  if (guided && e->cfg.cond_mode == B200MDM_COND_NONE)
    return fail(B200MDM_EINVAL, "classifier-free guidance needs a conditioned model (sampler_util.py:29)");
  TRY(check_seq_len(e, nframes + 1));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  TRY(select_workspace(e, slots, nframes, guided ? 2 : 1, s));
  TRY(ensure_slots(e));
  slots_reset_kernel<<<(e->Bp + 127) / 128, 128, 0, s>>>(e->slots, e->tvec, e->kvlen, e->scale,
                                                         e->cfg.cond_mode == B200MDM_COND_ACTION ? e->action : nullptr,
                                                         e->tmap, e->B, e->Bp, e->S);
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaMemsetAsync(e->x_work, 0, static_cast<size_t>(e->B) * e->JF * e->T * sizeof(float), s));
  e->launches += 1;
  end_cond(e);
  e->slot_mode = true;
  e->slot_sampler = mode;
  e->slot_flags = (flags & B200MDM_FLAG_CLIP_DENOISED) | B200MDM_FLAG_PHILOX_NOISE;
  e->slot_busy.assign(e->B, 0);
  e->slot_left.assign(e->B, 0);
  return B200MDM_OK;
}

static int check_slot(const b200mdm_engine* e, int32_t slot) {
  if (!e) return fail(B200MDM_EINVAL, "null engine");
  if (!e->slot_mode) return fail(B200MDM_ESTATE, "no slot session (b200mdm_slots_begin)");
  if (slot < 0 || slot >= e->B) return fail(B200MDM_EINVAL, "slot %d outside [0, %d)", slot, e->B);
  return B200MDM_OK;
}

extern "C" int b200mdm_slot_admit(b200mdm_engine* e, int32_t slot, const float* cond_embed_dev, int64_t action,
                                  float scale, int64_t length, uint64_t seed, int64_t sample_index, void* stream) {
  TRY(check_slot(e, slot));
  if (e->dec && !e->dec_clip) return fail(B200MDM_EINVAL, "a token-memory session admits through b200mdm_chain_slot_admit");
  if (e->slot_busy[slot]) return fail(B200MDM_ESTATE, "slot %d holds a request that has not been read", slot);
  const int mode = e->cfg.cond_mode;
  if ((mode == B200MDM_COND_TEXT || e->dec_clip) && !cond_embed_dev)
    return fail(B200MDM_EINVAL, "a text-conditioned model needs the request's text embedding");
  if (mode == B200MDM_COND_ACTION && (action < 0 || action >= e->cfg.num_actions))
    return fail(B200MDM_EINVAL, "action index out of range");
  if (!std::isfinite(scale)) return fail(B200MDM_EINVAL, "scale must be finite");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  // valid keys as upload_kvlen_scale counts them: the timestep token, then `length` frames (length < 0: every frame)
  int kv = e->S;
  if (e->cfg.mask_frames && length >= 0 && e->T > 1) kv = static_cast<int>(std::min<int64_t>(length, e->T)) + 1;
  const size_t n = static_cast<size_t>(e->JF) * e->T;
  slot_admit_kernel<<<1, 1, 0, s>>>(e->slots, e->tvec, e->kvlen, e->scale, mode == B200MDM_COND_ACTION ? e->action : nullptr,
                                     e->tmap, slot, e->B, e->halves, e->n_steps - 1, static_cast<unsigned long long>(seed),
                                     static_cast<long long>(sample_index), scale, kv, static_cast<int>(action));
  CUDA_TRY(cudaGetLastError());
  // x_T as p_sample_loop(noise_seed=seed) draws it for global sample `sample_index`
  TRY(launch_philox(e->x_work + slot * n, 1, static_cast<long long>(n), seed, sample_index, 0xffffffffu, nullptr, s));
  e->launches += 2;
  TRY(fill_condproj(e, cond_embed_dev, false, e->B, s, slot));
  if (e->dec_clip) TRY(cross_rows_per_sample(e, nullptr, s));
  e->slot_busy[slot] = 1;
  e->slot_left[slot] = e->n_steps;
  return B200MDM_OK;
}

extern "C" int b200mdm_slots_run(b200mdm_engine* e, int32_t n_steps, int32_t use_graph, void* stream) {
  if (!e) return fail(B200MDM_EINVAL, "null engine");
  if (!e->slot_mode) return fail(B200MDM_ESTATE, "no slot session (b200mdm_slots_begin)");
  if (n_steps <= 0) return fail(B200MDM_EINVAL, "n_steps %d <= 0", n_steps);
  TRY(check_ready(e, true));
  TRY(refuse(e, FAM_SLOTS));
  StepArgs a = loop_args(e, e->slot_sampler, 0, e->slot_flags, true);
  a.explicit_t = true;
  a.slots = true;
  cudaStream_t user = static_cast<cudaStream_t>(stream), s;
  TRY(loop_enter(e, a, e->slot_flags, use_graph, user, &s));
  for (int k = 0; k < n_steps; ++k) TRY(enqueue_step(e, a, s, use_graph));
  for (int b = 0; b < e->B; ++b) e->slot_left[b] = std::max(0, e->slot_left[b] - n_steps);
  return loop_leave(e, use_graph, user);
}

extern "C" int b200mdm_slot_read(b200mdm_engine* e, int32_t slot, float* out_dev, void* stream) {
  TRY(check_slot(e, slot));
  if (e->dec && !e->dec_clip) return fail(B200MDM_EINVAL, "a token-memory session reads through b200mdm_chain_slot_handoff");
  if (!out_dev) return fail(B200MDM_EINVAL, "null tensor");
  if (!e->slot_busy[slot] || e->slot_left[slot] > 0)
    return fail(B200MDM_ESTATE, "slot %d has no finished request (%d steps to run)", slot, e->slot_left[slot]);
  const size_t n = static_cast<size_t>(e->JF) * e->T;
  CUDA_TRY(cudaMemcpyAsync(out_dev, e->x_work + slot * n, n * sizeof(float), cudaMemcpyDeviceToDevice,
                           static_cast<cudaStream_t>(stream)));
  e->slot_busy[slot] = 0;
  return B200MDM_OK;
}

// ------------------------------------------------------------------------------------------------ DDIM inversion
// ddim_reverse_sample at schedule indices first_index, first_index+1, ... (n_run of them) on the engine's working
// buffer: the loop of b200mdm_sample_loop_range with the reverse epilogue, no noise and an upward step counter.
extern "C" int b200mdm_ddim_reverse_loop_range(b200mdm_engine* e, int32_t first_index, int32_t n_run, const float* x_in_dev,
                                               float* x_out_dev, int32_t flags, int32_t use_graph, void* stream) {
  TRY(check_flags("DDIM inversion", flags, B200MDM_FLAG_CLIP_DENOISED));
  if (n_run <= 0 || first_index < 0) return fail(B200MDM_EINVAL, "bad step range");
  TRY(check_ready(e, true));
  if (n_run > e->n_steps - first_index) return fail(B200MDM_EINVAL, "bad step range");
  TRY(need_table(e, TAB_NEXT));
  TRY(refuse(e, FAM_REVERSE));
  return run_loop(e, loop_args(e, B200MDM_MODE_DDIM_REVERSE, 0, flags, false), flags, first_index, n_run, x_in_dev, x_out_dev,
                  nullptr, 0, use_graph, stream);
}

// ------------------------------------------------------------------------------------------------ PLMS
static int ensure_plms(b200mdm_engine* e) {
  const size_t n = static_cast<size_t>(e->B) * e->JF * e->T;
  return alloc_all({{&e->plms_ring, PLMS_RING * n}, {&e->plms_mid, n}, {&e->plms_pred, n}});
}

extern "C" int b200mdm_plms_loop_range(b200mdm_engine* e, int32_t order, int32_t first_index, int32_t n_run,
                                       const float* x_in_dev, float* x_out_dev, int32_t flags, int32_t use_graph,
                                       void* stream) {
  if (order < 1 || order > 4) return fail(B200MDM_EINVAL, "PLMS order %d is not an integer from 1 to 4", order);
  TRY(check_flags("PLMS", flags, B200MDM_FLAG_CLIP_DENOISED));
  if (x_in_dev && order == 1)
    return fail(B200MDM_EINVAL, "a PLMS loop of order 1 has no first step (the reference needs old_out there)");
  if (n_run <= 0) return fail(B200MDM_EINVAL, "bad step range");
  TRY(check_ready(e, true));
  TRY(check_range_down(e, first_index, n_run));
  if (!x_in_dev && (e->plms_done < 0 || e->plms_order != order))
    return fail(B200MDM_ESTATE, "no PLMS loop of order %d to continue (pass x_in_dev)", order);
  TRY(refuse(e, FAM_PLMS));
  TRY(ensure_plms(e));
  // every step after the improved-Euler one is an Adams-Bashforth step: the launches of a DDIM step, one graph per order
  const int done = x_in_dev ? 0 : e->plms_done;
  return run_loop(e, loop_args(e, MODE_PLMS_AB, order, flags, false), flags, first_index, n_run, x_in_dev, x_out_dev, nullptr, 0,
                  use_graph, stream, done, done == 0);
}

extern "C" int b200mdm_plms_step(b200mdm_engine* e, int32_t index, int32_t order, const float* x_t_dev,
                                 const float* const* old_eps_dev, int32_t n_old, int32_t flags, float* x_out_dev,
                                 float* pred_xstart_dev, float* eps_out_dev, void* stream) {
  if (order < 1 || order > 4) return fail(B200MDM_EINVAL, "PLMS order %d is not an integer from 1 to 4", order);
  TRY(check_flags("PLMS", flags, B200MDM_FLAG_CLIP_DENOISED));
  // old_eps_dev NULL = no old_out (the improved-Euler step); non-NULL = old_out['old_eps'], which may be empty: the
  // reference then takes the Adams-Bashforth branch at cur_order 1 (gaussian_diffusion.py:1042-1056)
  const bool euler = old_eps_dev == nullptr;
  if (n_old < 0 || (euler && n_old != 0))
    return fail(B200MDM_EINVAL, "bad eps history (n_old %d with %s array)", n_old, euler ? "a null" : "an");
  if (euler && order == 1)
    return fail(B200MDM_EINVAL, "PLMS of order 1 needs an eps history (the reference needs old_out there)");
  if (!x_t_dev || !x_out_dev) return fail(B200MDM_EINVAL, "null tensor");
  const int h = n_old < PLMS_RING ? n_old : PLMS_RING;   // the newest h entries are all AB4 can use
  for (int j = 0; j < h; ++j)
    if (!old_eps_dev[n_old - h + j]) return fail(B200MDM_EINVAL, "null eps history entry %d", n_old - h + j);
  TRY(check_ready(e, true));
  if (index < 0 || index >= e->n_steps) return fail(B200MDM_EINVAL, "schedule index out of range");
  TRY(refuse(e, FAM_PLMS));
  TRY(ensure_plms(e));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t n = static_cast<size_t>(e->B) * e->JF * e->T, x_bytes = n * sizeof(float);
  // the history goes into ring slots 0..h-1, oldest first, as a loop that had made h evaluations would hold it
  for (int j = 0; j < h; ++j)
    CUDA_TRY(cudaMemcpyAsync(e->plms_ring + j * n, old_eps_dev[n_old - h + j], x_bytes, cudaMemcpyDeviceToDevice, s));
  step_set_kernel<<<1, 1, 0, s>>>(e->state, h, index, nullptr, 0, e->noise_seed, e->noise_sample_base, e->n_steps);
  CUDA_TRY(cudaGetLastError());
  e->launches += 1;
  e->plms_done = -1;
  StepArgs a;
  a.order = order;
  a.clip = (flags & B200MDM_FLAG_CLIP_DENOISED) ? 1 : 0;
  if (euler) {
    TRY(enqueue_plms_euler(e, a, x_t_dev, x_out_dev, s));
    if (pred_xstart_dev) CUDA_TRY(cudaMemcpyAsync(pred_xstart_dev, e->plms_pred, x_bytes, cudaMemcpyDeviceToDevice, s));
  } else {
    a.mode = MODE_PLMS_AB;
    a.x_in = x_t_dev;
    a.x_out = x_out_dev;
    a.pred = pred_xstart_dev;
    int nk = 0;
    TRY(enqueue_forward(e, a, s, &nk));
    e->launches += nk;
  }
  if (eps_out_dev)
    CUDA_TRY(cudaMemcpyAsync(eps_out_dev, e->plms_ring + (h % PLMS_RING) * n, x_bytes, cudaMemcpyDeviceToDevice, s));
  return B200MDM_OK;
}

// ------------------------------------------------------------------------------------------------ DPM-Solver++
static int ensure_dpm(b200mdm_engine* e) {
  return alloc_all({{&e->dpm_hist, DPM_SLOTS * static_cast<size_t>(e->B) * e->JF * e->T}});
}

// Multistep DPM-Solver++ (data prediction) at schedule indices first_index, first_index-1, ... (n_run of them) on the
// engine's working buffer: the launches of a DDIM step without the noise draw, one graph per order.  The step counter
// k = StepState::done selects the history slots and the first-order first step.
extern "C" int b200mdm_dpm_loop_range(b200mdm_engine* e, int32_t order, int32_t first_index, int32_t n_run,
                                      const float* x_in_dev, float* x_out_dev, int32_t flags, int32_t use_graph,
                                      void* stream) {
  if (order < 1 || order > 2) return fail(B200MDM_EINVAL, "DPM-Solver++ order %d is not 1 or 2", order);
  TRY(check_flags("DPM-Solver++", flags, B200MDM_FLAG_CLIP_DENOISED));
  if (n_run <= 0) return fail(B200MDM_EINVAL, "bad step range");
  TRY(check_ready(e, true));
  TRY(check_range_down(e, first_index, n_run));
  TRY(need_table(e, TAB_DPM));
  if (!x_in_dev && (e->dpm_done < 0 || e->dpm_order != order))
    return fail(B200MDM_ESTATE, "no DPM-Solver++ loop of order %d to continue (pass x_in_dev)", order);
  TRY(refuse(e, FAM_DPM));
  TRY(ensure_dpm(e));
  const int done = x_in_dev ? 0 : e->dpm_done;
  return run_loop(e, loop_args(e, MODE_DPM, order, flags, false), flags, first_index, n_run, x_in_dev, x_out_dev, nullptr, 0,
                  use_graph, stream, done);
}

extern "C" int b200mdm_dpm_pred_xstart(b200mdm_engine* e, float* out_dev, void* stream) {
  if (!e || !out_dev) return fail(B200MDM_EINVAL, "null argument");
  if (e->dpm_done <= 0 || !e->dpm_hist) return fail(B200MDM_ESTATE, "no DPM-Solver++ loop has run a step");
  const size_t n = static_cast<size_t>(e->B) * e->JF * e->T;
  CUDA_TRY(cudaMemcpyAsync(out_dev, e->dpm_hist + static_cast<size_t>((e->dpm_done - 1) & 1) * n, n * sizeof(float),
                           cudaMemcpyDeviceToDevice, static_cast<cudaStream_t>(stream)));
  return B200MDM_OK;
}

// ------------------------------------------------------------------------------------------------ autoregressive chain
template <class T>
static int ensure_cap(T** p, size_t* cap, size_t n) {
  if (*cap >= n) return B200MDM_OK;
  dfree(*p);
  *cap = 0;
  TRY(dalloc(p, n));
  *cap = n;
  return B200MDM_OK;
}

// DiP's chain of prefix completions (AutoRegressiveSampler) as one engine loop: the layout, and every chunk's memory
// projected once, here.
extern "C" int b200mdm_chain_setup(b200mdm_engine* e, int32_t n_chunks, int32_t pred_len, int32_t context_len,
                                   int32_t include_prefix, int32_t crop, const float* enc_chunks_dev,
                                   const uint8_t* text_mask_chunks_host, void* stream) {
  if (!e) return fail(B200MDM_EINVAL, "null engine");
  if (n_chunks <= 0) return fail(B200MDM_EINVAL, "n_chunks %d <= 0", n_chunks);
  if (pred_len <= 0 || context_len <= 0 || context_len > pred_len)
    return fail(B200MDM_EINVAL, "pred_len %d / context_len %d: a chunk hands on 1 .. pred_len frames", pred_len, context_len);
  const long long total = (include_prefix ? context_len : 0) + static_cast<long long>(n_chunks) * pred_len;
  if (crop <= 0 || crop > total) return fail(B200MDM_EINVAL, "crop %d outside the chain's 1 .. %lld frames", crop, total);
  if ((enc_chunks_dev == nullptr) != (text_mask_chunks_host == nullptr))
    return fail(B200MDM_EINVAL, "per-chunk memories need both the token features and the masks");
  if (!is_prefix_engine(e)) return fail(B200MDM_EINVAL, "the chain is for prefix-completion (DiP) engines");
  if (!e->finalized || !e->cond_set || !e->prefix_set)
    return fail(B200MDM_ESTATE, "weights, b200mdm_set_cond_dec and b200mdm_set_prefix first");
  if (pred_len != e->T || context_len != e->ctx)
    return fail(B200MDM_EINVAL, "pred_len %d / context_len %d differ from the conditioning's %d / the model's %d", pred_len,
                context_len, e->T, e->ctx);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int B = e->B, Bp = e->Bp, Mt = e->Mt, d = e->d, C = e->cfg.cond_dim;
  e->chain_next = -1;
  if (e->chain_prefix_cap < static_cast<size_t>(B) * e->JF * e->ctx || (enc_chunks_dev && e->chain_mem_cap < static_cast<size_t>(n_chunks) * Bp * Mt * d)) {
    CUDA_TRY(cudaDeviceSynchronize());   // a previous chain may still read the buffers being replaced
  }
  TRY(ensure_cap(&e->chain_prefix, &e->chain_prefix_cap, static_cast<size_t>(B) * e->JF * e->ctx));
  e->chain_mems = enc_chunks_dev != nullptr;
  if (e->chain_mems) {
    const size_t mem = static_cast<size_t>(Bp) * Mt * d, msk = static_cast<size_t>(Bp) * Mt;
    TRY(ensure_cap(&e->chain_mem, &e->chain_mem_cap, n_chunks * mem));
    TRY(ensure_cap(&e->chain_mask, &e->chain_mask_cap, n_chunks * msk));
    std::vector<unsigned char>& mk = e->h_chain_mask;   // staged in the engine until the next call, as b200mdm_set_cond_dec's
    mk.resize(n_chunks * msk);
    for (int c = 0; c < n_chunks; ++c)
      pack_text_mask(mk.data() + c * msk, text_mask_chunks_host + static_cast<size_t>(c) * B * Mt, 1, B, Bp, Mt);
    CUDA_TRY(cudaMemcpyAsync(e->chain_mask, mk.data(), mk.size(), cudaMemcpyHostToDevice, s));
    // each chunk's text_emb, as b200mdm_set_cond_dec projects one
    for (int c = 0; c < n_chunks; ++c)
      TRY(build_text_memory(e, enc_chunks_dev + static_cast<size_t>(c) * Mt * B * C, 1, e->mem_uncond, e->chain_mem + c * mem, s));
  }
  e->chain_n = n_chunks;
  e->goal_set = false;
  e->chain_off = include_prefix ? context_len : 0;
  e->chain_crop = crop;
  e->chain_next = 0;
  return B200MDM_OK;
}

// ---- goal-directed chains (chunk_frame.cuh)
static int check_chunk_frame(const void* carry, const void* frames, int B, int D, int n, const void* mean, const void* std,
                             const void* goal, int n_ext, const void* target) {
  if (!carry || (!frames && n > 0) || !mean || !std || !goal || !target) return fail(B200MDM_EINVAL, "null argument");
  if (B <= 0 || D < 4 || n < 0 || n > JG_MAX_FRAMES || n_ext < 2 || n_ext > 64)
    return fail(B200MDM_EINVAL, "batch %d, %d features, %d frames, %d goal entries: batch >= 1, >= 4 features, 0 .. %d frames "
                "and 2 .. 64 entries", B, D, n, n_ext, JG_MAX_FRAMES);
  return B200MDM_OK;
}
static int launch_chunk_frame(double* carry, const float* frames, int B, int D, int n, const float* mean, const float* std,
                              const float* goal, int n_ext, float* target, cudaStream_t s) {
  chunk_frame_kernel<<<B, JG_THREADS, 0, s>>>(frames, D, n, mean, std, carry, goal, n_ext, target);
  CUDA_TRY(cudaGetLastError());
  return B200MDM_OK;
}
// chunk c's goal rows [B, n_ext, 3]: one goal for the whole chain, or one per chunk
static const float* goal_row(const b200mdm_engine* e, int c) {
  return e->goal_src + (e->goal_n == 1 ? 0 : static_cast<size_t>(c) * e->B * e->cfg.target_joints * 3);
}

extern "C" int b200mdm_chunk_frame(double* carry_dev, const float* frames_dev, int32_t batch, int32_t n_feats,
                                   int32_t n_frames, const float* mean_dev, const float* std_dev, const float* goal_dev,
                                   int32_t n_ext, float* target_dev, void* stream) {
  TRY(check_chunk_frame(carry_dev, frames_dev, batch, n_feats, n_frames, mean_dev, std_dev, goal_dev, n_ext, target_dev));
  return launch_chunk_frame(carry_dev, frames_dev, batch, n_feats, n_frames, mean_dev, std_dev, goal_dev, n_ext, target_dev,
                            static_cast<cudaStream_t>(stream));
}

// Goals for the chain set up last: chunk 0's carry (over the prefix under include_prefix, else none) and target, then
// its embedding into the workspace's target, which every step graph of the chain reads.
extern "C" int b200mdm_chain_set_goal(b200mdm_engine* e, const float* mean_dev, const float* std_dev, const float* goal_dev,
                                      int32_t n_goals, const uint8_t* valid_host, void* stream) {
  if (!e) return fail(B200MDM_EINVAL, "null engine");
  if (!mean_dev || !std_dev || !goal_dev || !valid_host) return fail(B200MDM_EINVAL, "null argument");
  if (e->cfg.target_encoder == B200MDM_TARGET_NONE) return fail(B200MDM_EINVAL, "this engine has no target encoder");
  if (!is_prefix_engine(e)) return fail(B200MDM_EINVAL, "the chain is for prefix-completion (DiP) engines");
  if (e->chain_next != 0) return fail(B200MDM_ESTATE, "b200mdm_chain_setup first (a goal is set before the chain runs)");
  if (n_goals != 1 && n_goals != e->chain_n)
    return fail(B200MDM_EINVAL, "%d goals: one for the whole chain or one per chunk (%d)", n_goals, e->chain_n);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int B = e->B, n_ext = e->cfg.target_joints;
  if (e->goal_carry_cap < static_cast<size_t>(B) * CF_CARRY || e->goal_tgt_cap < static_cast<size_t>(B) * n_ext * 3) {
    CUDA_TRY(cudaDeviceSynchronize());   // a previous chain may still read the buffers being replaced
  }
  TRY(ensure_cap(&e->goal_carry, &e->goal_carry_cap, static_cast<size_t>(B) * CF_CARRY));
  TRY(ensure_cap(&e->goal_tgt, &e->goal_tgt_cap, static_cast<size_t>(B) * n_ext * 3));
  e->goal_mean = mean_dev;
  e->goal_std = std_dev;
  e->goal_src = goal_dev;
  e->goal_n = n_goals;
  CUDA_TRY(cudaMemsetAsync(e->goal_carry, 0, static_cast<size_t>(B) * CF_CARRY * sizeof(double), s));
  TRY(launch_chunk_frame(e->goal_carry, e->prefix_src, B, e->JF, e->chain_off, mean_dev, std_dev, goal_row(e, 0), n_ext,
                         e->goal_tgt, s));
  TRY(encode_target(e, e->goal_tgt, valid_host, B, e->tgt_valid, e->tgt_g, e->h_valid, s));
  e->launches += 2;
  e->target_set = true;
  e->goal_set = true;
  return B200MDM_OK;
}

// Global steps first_step .. first_step + n_run - 1 of the chain; step k is step k % N of chunk k / N (N = n_steps).  A
// chunk starts with its memory and x_T in x_work and the step state reset (cur = N - 1, done = 0), so one step graph
// serves every step of every chunk; after its last step chain_handoff_kernel writes the sample to the output and hands
// its last ctx frames on as the next chunk's prefix.
extern "C" int b200mdm_chain_loop_range(b200mdm_engine* e, int32_t mode, int32_t order, int32_t first_step, int32_t n_run,
                                        const float* x_T_dev, int64_t x_T_chunk_stride, const float* noise_tape_dev,
                                        int64_t noise_step_stride, float* out_dev, int32_t flags, int32_t use_graph,
                                        void* stream) {
  if (!e) return fail(B200MDM_EINVAL, "null engine");
  const bool dpm = mode == MODE_DPM;
  if (mode != B200MDM_MODE_DDPM && mode != B200MDM_MODE_DDIM && !dpm)
    return fail(B200MDM_EINVAL, "chain mode %d: B200MDM_MODE_DDPM, B200MDM_MODE_DDIM or 7 (DPM-Solver++)", mode);
  if (dpm ? (order < 1 || order > 2) : order != 0)
    return fail(B200MDM_EINVAL, "order %d: 1 or 2 for DPM-Solver++, 0 otherwise", order);
  TRY(check_flags("a chain", flags, B200MDM_FLAG_CLIP_DENOISED | B200MDM_FLAG_PHILOX_NOISE));
  const bool philox = (flags & B200MDM_FLAG_PHILOX_NOISE) != 0;
  if (!philox && (!x_T_dev || (!dpm && !noise_tape_dev)))
    return fail(B200MDM_EINVAL, "null x_T or noise tape (or pass B200MDM_FLAG_PHILOX_NOISE)");
  if (!out_dev) return fail(B200MDM_EINVAL, "null output");
  if (first_step < 0 || n_run <= 0) return fail(B200MDM_EINVAL, "bad step range");
  if (!is_prefix_engine(e)) return fail(B200MDM_EINVAL, "the chain is for prefix-completion (DiP) engines");
  if (e->n_steps <= 0) return fail(B200MDM_ESTATE, "b200mdm_set_schedule has not been called");
  if (dpm) TRY(need_table(e, TAB_DPM));
  if (e->chain_next < 0 || first_step != e->chain_next)
    return fail(B200MDM_ESTATE, "no chain to run from step %d (b200mdm_chain_setup; next step %d)", first_step, e->chain_next);
  const int N = e->n_steps;
  if (static_cast<long long>(first_step) + n_run > static_cast<long long>(e->chain_n) * N)
    return fail(B200MDM_EINVAL, "steps %d .. %d past the chain's %d x %d", first_step, first_step + n_run - 1, e->chain_n, N);
  if (dpm) TRY(ensure_dpm(e));
  const bool goal = e->goal_set;
  const StepArgs a = loop_args(e, mode, order, flags, philox && !dpm);
  cudaStream_t user = static_cast<cudaStream_t>(stream), s;
  TRY(loop_enter(e, a, flags, use_graph, user, &s));
  // The chain consumes the conditioning: it replaces the memory (per-chunk memories) and the prefix rows, so every
  // other call needs b200mdm_set_cond_dec and b200mdm_set_prefix again (chain_next, not cond_set, admits its own calls).
  e->cond_set = false;
  e->prefix_set = false;
  const int B = e->B, JF = e->JF, T = e->T;
  const size_t n = static_cast<size_t>(B) * JF * T, mem = static_cast<size_t>(e->Bp) * e->Mt * e->d,
               msk = static_cast<size_t>(e->Bp) * e->Mt;
  for (int k = first_step; k < first_step + n_run; ++k) {
    const int c = k / N, j = k % N;
    if (j == 0) {
      if (e->chain_mems) {
        CUDA_TRY(cudaMemcpyAsync(e->memproj, e->chain_mem + c * mem, mem * sizeof(float), cudaMemcpyDeviceToDevice, s));
        CUDA_TRY(cudaMemcpyAsync(e->memmask, e->chain_mask + c * msk, msk, cudaMemcpyDeviceToDevice, s));
      }
      if (x_T_dev) {
        CUDA_TRY(cudaMemcpyAsync(e->x_work, x_T_dev + c * x_T_chunk_stride, n * sizeof(float), cudaMemcpyDeviceToDevice, s));
      } else {   // the x_T of b200mdm_philox_normal(step_id -1): the same for every chunk, as the host chain draws it
        TRY(launch_philox(e->x_work, B, static_cast<long long>(JF) * T, e->noise_seed, e->noise_sample_base, 0xffffffffu,
                          nullptr, s));
        e->launches += 1;
      }
    }
    if (j == 0 || k == first_step) {
      // DPM-Solver++ counts its steps within the chunk (first-order first step, history slots); the noise tape of the
      // DDPM / DDIM step k is at + (k - first_step) * stride of this call's tape
      const float* tape = noise_tape_dev && !philox ? noise_tape_dev + static_cast<long long>(k - first_step) * noise_step_stride : nullptr;
      step_set_kernel<<<1, 1, 0, s>>>(e->state, dpm ? j : 0, N - 1 - j, tape, noise_step_stride, e->noise_seed,
                                      e->noise_sample_base, N);
      CUDA_TRY(cudaGetLastError());
      e->launches += 1;
    }
    TRY(enqueue_step(e, a, s, use_graph));
    if (j == N - 1) {
      const bool last = c == e->chain_n - 1;
      const long long rows = static_cast<long long>(B) * JF;
      chain_handoff_kernel<<<static_cast<int>((rows * T + 255) / 256 < 1184 ? (rows * T + 255) / 256 : 1184), 256, 0, s>>>(
          e->x_work, out_dev, last ? nullptr : e->chain_prefix, rows, T, e->ctx, e->chain_off + c * T, e->chain_crop);
      CUDA_TRY(cudaGetLastError());
      e->launches += 1;
      if (!last) {
        TRY(launch_pack_input(e->chain_prefix, e->xin16, B, JF, e->ctx, e->S, e->Kp_in, 0, s));
        e->launches += 1;
      }
      if (!last && goal) {   // chunk c + 1's target, in its own frame, into the embedding the step graph reads
        TRY(launch_chunk_frame(e->goal_carry, e->x_work, B, JF, T, e->goal_mean, e->goal_std, goal_row(e, c + 1),
                               e->cfg.target_joints, e->goal_tgt, s));
        TRY(embed_target(e, e->goal_tgt, e->tgt_valid, B, e->tgt_g, s));
        e->launches += 2;
      }
    }
  }
  const int next = first_step + n_run;
  e->chain_next = next < e->chain_n * N ? next : -1;
  return loop_leave(e, use_graph, user);
}

// ------------------------------------------------------------------------------------------------ token-memory slots
// DESIGN.md, "Continuous batching", "Token memories and chains": DiP's chains and the plain BERT decoder in slots.  The
// step graph is the slot graph of b200mdm_slots_begin; what is per slot here -- the memory rows (memproj, memmask), the
// prefix rows of the embedding GEMM's A operand and the chunk position -- is written between replays, on the stream, by
// the host, which knows every chunk boundary without asking the device.
extern "C" int b200mdm_chain_slots_begin(b200mdm_engine* e, int32_t slots, int32_t nframes, int32_t guided, int32_t mode,
                                         int32_t flags, int32_t n_tokens, void* stream) {
  if (!e) return fail(B200MDM_EINVAL, "null engine");
  if (!e->finalized) return fail(B200MDM_ESTATE, "weights not finalised");
  if (e->n_steps <= 0) return fail(B200MDM_ESTATE, "b200mdm_set_schedule has not been called");
  if (!e->dec || e->dec_clip)
    return fail(B200MDM_EINVAL, "b200mdm_chain_slots_begin is for BERT-memory decoders (the others: b200mdm_slots_begin)");
  if (slots <= 0 || nframes <= 0) return fail(B200MDM_EINVAL, "bad slots / nframes");
  if (n_tokens <= 0 || n_tokens > XAL_MAX_MT)
    return fail(B200MDM_EINVAL, "n_tokens %d: a text memory holds 1..%d tokens (DistilBERT's position limit)", n_tokens,
                XAL_MAX_MT);
  if (mode != B200MDM_MODE_DDPM && mode != B200MDM_MODE_DDIM)
    return fail(B200MDM_ENOTIMPL, "continuous batching runs DDPM and DDIM (PLMS, DPM-Solver++, DDIM inversion and the "
                "bound carry history or tables that are not per slot)");
  if (flags & B200MDM_FLAG_CONST_NOISE) return fail(B200MDM_ENOTIMPL, "B200MDM_FLAG_CONST_NOISE with continuous batching");
  TRY(check_flags("continuous batching", flags, B200MDM_FLAG_CLIP_DENOISED | B200MDM_FLAG_PHILOX_NOISE));
  TRY(check_seq_len(e, nframes + e->ctx));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  TRY(select_workspace(e, slots, nframes, guided ? 2 : 1, s));
  TRY(ensure_slots(e));
  TRY(ensure_text_memory(e, n_tokens));   // the one place the memory is sized: admissions never resize it
  if (e->ctx > 0) {
    const size_t np = static_cast<size_t>(e->B) * e->JF * e->ctx;
    if (e->chain_prefix_cap < np) CUDA_TRY(cudaDeviceSynchronize());   // a chain may still read the buffer being replaced
    TRY(ensure_cap(&e->chain_prefix, &e->chain_prefix_cap, np));
  }
  slots_reset_kernel<<<(e->Bp + 127) / 128, 128, 0, s>>>(e->slots, e->tvec, e->kvlen, e->scale, nullptr, e->tmap, e->B,
                                                         e->Bp, e->S);
  CUDA_TRY(cudaGetLastError());
  // every memory row the unconditional one (W 0 + b) without padding: what an idle slot attends, and for good the rows
  // of the unconditional half, which an admission leaves as they are
  memproj_group_fill_kernel<<<dim3(e->Mt, e->Bp), 128, 0, s>>>(e->memproj, e->memtok, e->b_txt, 0, e->Mt, e->d);
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaMemsetAsync(e->memmask, 0, static_cast<size_t>(e->Bp) * e->Mt, s));
  CUDA_TRY(cudaMemsetAsync(e->x_work, 0, static_cast<size_t>(e->B) * e->JF * e->T * sizeof(float), s));
  e->launches += 2;
  end_cond(e);
  e->mem_uncond = false;
  e->prefix_set = e->ctx > 0;   // each slot packs its own prefix rows
  e->prefix_src = nullptr;
  e->slot_mode = true;
  e->slot_sampler = mode;
  e->slot_flags = (flags & B200MDM_FLAG_CLIP_DENOISED) | B200MDM_FLAG_PHILOX_NOISE;
  e->slot_busy.assign(e->B, 0);
  e->slot_left.assign(e->B, 0);
  e->chain_slot.assign(e->B, b200mdm_engine::ChainSlot{});
  return B200MDM_OK;
}

static int check_token_slot(const b200mdm_engine* e, int32_t slot) {
  TRY(check_slot(e, slot));
  if (!e->dec || e->dec_clip) return fail(B200MDM_EINVAL, "not a token-memory session (b200mdm_chain_slots_begin)");
  return B200MDM_OK;
}
// Slot b's conditional memory rows W tokens + b (tokens [Mt, C]: memproj rows b * Mt .., as build_text_memory projects
// sample b's) and its mask rows in every half: 2 launches.
static int slot_memory(b200mdm_engine* e, int slot, const float* tokens, const uint8_t* mask, cudaStream_t s) {
  const int d = e->d, Mt = e->Mt, C = e->cfg.cond_dim;
  const size_t warps = static_cast<size_t>(Mt) * d;
  small_linear_kernel<0><<<static_cast<int>((warps * 32 + 255) / 256), 256, 0, s>>>(
      tokens, e->w_txt, e->b_txt, e->memproj + static_cast<size_t>(slot) * Mt * d, Mt, d, C, C);
  CUDA_TRY(cudaGetLastError());
  slot_mask_kernel<<<1, 128, 0, s>>>(e->memmask, mask, slot, e->B, e->halves, Mt);
  CUDA_TRY(cudaGetLastError());
  e->launches += 2;
  return B200MDM_OK;
}
// prefix [JF, ctx] into the first ctx rows of slot b's sequence of the embedding GEMM's A operand: 1 launch
static int slot_prefix(b200mdm_engine* e, int slot, const float* prefix, cudaStream_t s) {
  TRY(launch_pack_input(prefix, e->xin16 + static_cast<size_t>(slot) * e->S * 3 * e->Kp_in, 1, e->JF, e->ctx, e->S, e->Kp_in, 0,
                        s));
  e->launches += 1;
  return B200MDM_OK;
}
// Slot b at schedule index n_steps - 1 with its key, scale and key counts, and its x_T (step id -1 of its Philox
// stream, as p_sample_loop(noise_seed=seed) draws it for that sample): 2 launches.
static int slot_arm(b200mdm_engine* e, int slot, const b200mdm_engine::ChainSlot& r, cudaStream_t s) {
  const size_t n = static_cast<size_t>(e->JF) * e->T;
  slot_admit_kernel<<<1, 1, 0, s>>>(e->slots, e->tvec, e->kvlen, e->scale, nullptr, e->tmap, slot, e->B, e->halves,
                                     e->n_steps - 1, r.seed, r.g, r.scale, r.kv, 0);
  CUDA_TRY(cudaGetLastError());
  TRY(launch_philox(e->x_work + slot * n, 1, static_cast<long long>(n), r.seed, r.g, 0xffffffffu, nullptr, s));
  e->launches += 2;
  return B200MDM_OK;
}

extern "C" int b200mdm_chain_slot_admit(b200mdm_engine* e, int32_t slot, const float* tokens_dev, const uint8_t* mask_dev,
                                        const float* prefix_dev, float scale, int64_t length, int32_t include_prefix,
                                        uint64_t seed, int64_t sample_index, void* stream) {
  TRY(check_token_slot(e, slot));
  if (e->slot_busy[slot]) return fail(B200MDM_ESTATE, "slot %d holds a request", slot);
  if (!tokens_dev || !mask_dev) return fail(B200MDM_EINVAL, "the request's tokens and mask are required");
  if ((prefix_dev != nullptr) != (e->ctx > 0))
    return fail(B200MDM_EINVAL, "a prefix [njoints * nfeats, %d] for DiP, none for the plain BERT decoder", e->ctx);
  if (length < 1 || length > (1 << 24) || (e->ctx == 0 && length > e->T))
    return fail(B200MDM_EINVAL, "length %lld: 1 .. %d frames", static_cast<long long>(length), e->ctx == 0 ? e->T : 1 << 24);
  if (!std::isfinite(scale)) return fail(B200MDM_EINVAL, "scale must be finite");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  b200mdm_engine::ChainSlot r;
  r.seed = static_cast<unsigned long long>(seed);
  r.g = static_cast<long long>(sample_index);
  r.scale = scale;
  r.length = static_cast<int>(length);
  // valid keys: a DiP chunk attends all its ctx + pred_len frames (the length only crops the motion); the plain BERT
  // decoder has no token ahead of the frames, so `length` frames under mask_frames, as upload_kvlen_scale counts them
  r.kv = e->S;
  if (e->ctx == 0 && e->cfg.mask_frames && e->S > 1) r.kv = r.length;
  r.off = include_prefix && e->ctx > 0 ? e->ctx : 0;
  r.n_chunks = e->ctx > 0 ? (r.length + e->T - 1) / e->T : 1;
  TRY(slot_memory(e, slot, tokens_dev, mask_dev, s));
  if (e->ctx > 0) TRY(slot_prefix(e, slot, prefix_dev, s));
  TRY(slot_arm(e, slot, r, s));
  e->chain_slot[slot] = r;
  e->slot_busy[slot] = 1;
  e->slot_left[slot] = e->n_steps;
  return B200MDM_OK;
}

extern "C" int b200mdm_chain_slot_handoff(b200mdm_engine* e, int32_t slot, float* out_dev, const float* tokens_dev,
                                          const uint8_t* mask_dev, void* stream) {
  TRY(check_token_slot(e, slot));
  if (!out_dev) return fail(B200MDM_EINVAL, "null output");
  if ((tokens_dev == nullptr) != (mask_dev == nullptr)) return fail(B200MDM_EINVAL, "a new prompt needs its tokens and mask");
  if (!e->slot_busy[slot] || e->slot_left[slot] > 0)
    return fail(B200MDM_ESTATE, "slot %d has not just finished a chunk (%d steps to run)", slot,
                e->slot_busy[slot] ? e->slot_left[slot] : 0);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  b200mdm_engine::ChainSlot& r = e->chain_slot[slot];
  const bool last = r.chunk + 1 >= r.n_chunks;
  const int JF = e->JF, T = e->T;
  float* prefix = last ? nullptr : e->chain_prefix + static_cast<size_t>(slot) * JF * e->ctx;
  const long long rows = JF;
  chain_handoff_kernel<<<static_cast<int>((rows * T + 255) / 256 < 1184 ? (rows * T + 255) / 256 : 1184), 256, 0, s>>>(
      e->x_work + static_cast<size_t>(slot) * JF * T, out_dev, prefix, rows, T, e->ctx, r.off + r.chunk * T, r.length);
  CUDA_TRY(cudaGetLastError());
  e->launches += 1;
  if (last) {
    e->slot_busy[slot] = 0;
    return B200MDM_OK;
  }
  TRY(slot_prefix(e, slot, prefix, s));
  if (tokens_dev) TRY(slot_memory(e, slot, tokens_dev, mask_dev, s));
  TRY(slot_arm(e, slot, r, s));
  r.chunk += 1;
  e->slot_left[slot] = e->n_steps;
  return B200MDM_OK;
}

// ------------------------------------------------------------------------------------------------ variational bound
static int ensure_vb(b200mdm_engine* e) {
  const size_t n = static_cast<size_t>(e->B) * e->JF * e->T;
  if (e->vb_terms && e->vb_cap < e->n_steps) {   // a longer schedule: the step graph holds the old pointer
    drop_graph(e);
    dfree(e->vb_terms);
    e->vb_live = false;
  }
  const bool new_terms = !e->vb_terms;
  const int r = alloc_all({{&e->vb_xs, n},
                           {&e->vb_part, static_cast<size_t>(VB_TERMS) * e->B * e->T * ((e->JF + 31) / 32)},
                           {&e->vb_terms, static_cast<size_t>(VB_TERMS) * e->B * e->sched_cap}});
  if (r != B200MDM_OK) {
    e->vb_cap = 0;
    e->vb_live = false;
  } else if (new_terms) {
    e->vb_cap = e->sched_cap;
  }
  return r;
}

// The bound loop (calc_bpd_loop) at schedule indices first_index, first_index-1, ... (n_run of them): per step
// vb_xt_kernel, the forward with the EpiOut<OutVb> epilogue and vb_reduce_kernel, one graph.  The step state's `done`
// indexes this call's noise tape.
extern "C" int b200mdm_vb_loop_range(b200mdm_engine* e, int32_t first_index, int32_t n_run, const float* x_start_dev,
                                     const float* noise_tape_dev, int64_t noise_step_stride, int32_t flags,
                                     float* terms_dev, float* bpd_dev, int32_t use_graph, void* stream) {
  TRY(check_flags("the bound loop", flags, B200MDM_FLAG_CLIP_DENOISED | B200MDM_FLAG_PHILOX_NOISE));
  const bool philox = (flags & B200MDM_FLAG_PHILOX_NOISE) != 0;
  if (!philox && !noise_tape_dev) return fail(B200MDM_EINVAL, "null noise tape (or pass B200MDM_FLAG_PHILOX_NOISE)");
  if (n_run <= 0) return fail(B200MDM_EINVAL, "bad step range");
  TRY(check_ready(e, true));
  TRY(check_range_down(e, first_index, n_run));
  TRY(need_table(e, TAB_VB));
  if (!x_start_dev && !e->vb_live) return fail(B200MDM_ESTATE, "no bound loop to continue (pass x_start_dev)");
  TRY(refuse(e, FAM_VB));
  TRY(ensure_vb(e));
  if (!x_start_dev && !e->vb_live)   // ensure_vb reallocated the tables for a longer schedule: nothing to continue
    return fail(B200MDM_ESTATE, "the schedule outgrew the bound loop's tables: no bound loop to continue (pass x_start_dev)");
  cudaStream_t user = static_cast<cudaStream_t>(stream);
  const size_t n = static_cast<size_t>(e->B) * e->JF * e->T;
  if (x_start_dev) {   // a fresh loop: x_start in, every column of the tables cleared
    CUDA_TRY(cudaMemcpyAsync(e->vb_xs, x_start_dev, n * sizeof(float), cudaMemcpyDeviceToDevice, user));
    CUDA_TRY(cudaMemsetAsync(e->vb_terms, 0, static_cast<size_t>(VB_TERMS) * e->B * e->vb_cap * sizeof(float), user));
  }
  e->vb_live = true;
  TRY(run_loop(e, loop_args(e, MODE_VB, 0, flags, philox), flags, first_index, n_run, nullptr, nullptr, noise_tape_dev,
               noise_step_stride, use_graph, stream));
  if (terms_dev)
    CUDA_TRY(cudaMemcpy2DAsync(terms_dev, e->n_steps * sizeof(float), e->vb_terms, e->vb_cap * sizeof(float),
                               e->n_steps * sizeof(float), static_cast<size_t>(VB_TERMS) * e->B, cudaMemcpyDeviceToDevice, user));
  if (bpd_dev && first_index - n_run + 1 == 0) {
    vb_final_kernel<<<e->B, VB_REDUCE_THREADS, 0, user>>>(bpd_dev, e->vb_terms, e->vb_cap, e->vb_xs, e->tab[TAB_VB], e->n_steps,
                                                           e->B, e->JF * e->T);
    CUDA_TRY(cudaGetLastError());
    e->launches += 1;
  }
  return B200MDM_OK;
}

// Counter-based noise stream of the engine (Philox4x32-10 + Box-Muller, kernels.cuh): eps of schedule index i for
// global sample g depends on (seed, i, g, element) only -- not on the batch split, the GPU count or the chunking.
extern "C" int b200mdm_set_noise_stream(b200mdm_engine* e, uint64_t seed, int64_t sample_index_base) {
  if (!e) return fail(B200MDM_EINVAL, "null engine");
  e->noise_seed = seed;
  e->noise_sample_base = sample_index_base;
  return B200MDM_OK;
}
extern "C" int b200mdm_philox_normal(float* out_dev, int32_t batch, int64_t n_per_sample, uint64_t seed,
                                     int64_t sample_index_base, int32_t step_id, void* stream) {
  if (!out_dev || batch <= 0 || n_per_sample <= 0) return fail(B200MDM_EINVAL, "bad argument");
  return launch_philox(out_dev, batch, n_per_sample, seed, sample_index_base, static_cast<uint32_t>(step_id), nullptr,
                       static_cast<cudaStream_t>(stream));
}

extern "C" int b200mdm_q_sample(b200mdm_engine* e, float sqrt_ac, float sqrt_1mac, const float* x_start_dev,
                                const float* noise_dev, float* out_dev, int64_t n, void* stream) {
  if (!e || !noise_dev || !out_dev || n <= 0) return fail(B200MDM_EINVAL, "bad argument");
  q_sample_kernel<<<592, 256, 0, static_cast<cudaStream_t>(stream)>>>(out_dev, x_start_dev, noise_dev, sqrt_ac, sqrt_1mac,
                                                                     static_cast<size_t>(n));
  CUDA_TRY(cudaGetLastError());
  e->launches++;
  return B200MDM_OK;
}

extern "C" int64_t b200mdm_launch_count(b200mdm_engine* e, int32_t reset) {
  if (!e) return 0;
  long long v = e->launches;
  if (reset) e->launches = 0;
  return v;
}

// ------------------------------------------------------------------------------------------------ kernel tests
// What every GEMM test hook does before its launches: the kernels' attributes, and the SM count of the current device.
static int test_prologue(int* sms) {
  TRY(init_kernel_attrs());
  int dev = 0;
  CUDA_TRY(cudaGetDevice(&dev));
  CUDA_TRY(cudaDeviceGetAttribute(sms, cudaDevAttrMultiProcessorCount, dev));
  return B200MDM_OK;
}

extern "C" int b200mdm_test_gemm_f16(const void* a16_dev, const void* w16_dev, const float* bias_dev, void* out16_dev,
                                     int32_t M, int32_t N, int32_t K, int32_t act, int32_t block_n, void* stream) {
  if (!a16_dev || !w16_dev || !bias_dev || !out16_dev || M <= 0 || N <= 0 || K <= 0 || K % 8 || N % 8)
    return fail(B200MDM_EINVAL, "bad argument (K %% 8 == 0, N %% 8 == 0 required)");
  if (block_n != PP_BLOCK_N)
    return fail(B200MDM_EINVAL, "block_n must be 128 (the 128 x 128 tiles of the step's ping-pong projection kernel)");
  int sms = 132;
  TRY(test_prologue(&sms));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CUtensorMap ma, mb, mc;
  TRY(make_map(&ma, a16_dev, M, K, K, GEMM_BLOCK_M));
  TRY(make_map(&mb, w16_dev, N, K, K, PP_BLOCK_N));
  TRY(make_map_t(&mc, out16_dev, 2, M, N, N, 32));
  return act ? launch_gemm_bias<true>(ma, mb, mc, M, N, K, bias_dev, s, sms)
             : launch_gemm_bias<false>(ma, mb, mc, M, N, K, bias_dev, s, sms);
}

// Scratch device memory of a kernel-test entry point, allocated and freed in the order of `s`.
struct StreamScratch {
  cudaStream_t s;
  std::vector<void*> ptrs;
  explicit StreamScratch(cudaStream_t st) : s(st) {}
  ~StreamScratch() {
    for (void* p : ptrs) cudaFreeAsync(p, s);
  }
  template <class T>
  int alloc(T** p, size_t n, bool zero = false) {
    CUDA_TRY(cudaMallocAsync(reinterpret_cast<void**>(p), n * sizeof(T), s));
    ptrs.push_back(*p);
    if (zero) CUDA_TRY(cudaMemsetAsync(*p, 0, n * sizeof(T), s));
    return B200MDM_OK;
  }
};

extern "C" int b200mdm_test_gemm_epi(const void* a16_dev, const void* w16_dev, const float* bias_dev, void* out16_dev,
                                     int32_t M, int32_t N, int32_t K, int32_t epi, void* stream) {
  if (!a16_dev || !w16_dev || !bias_dev || !out16_dev || M <= 0 || N <= 0 || K <= 0 || K % 8)
    return fail(B200MDM_EINVAL, "bad argument (K %% 8 == 0 required)");
  int sms = 132;
  TRY(test_prologue(&sms));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CUtensorMap ma, mb, mc;
  TRY(make_map(&ma, a16_dev, M, K, K, GEMM_BLOCK_M));
  TRY(make_map(&mb, w16_dev, N, K, K, 128));
  if (epi == 0) {
    // the hi slab of the last 64-column block must not reach into the lo half: N % 64 == 0
    if (N % 64) return fail(B200MDM_EINVAL, "EpiBiasF16Wide needs N %% 64 == 0");
    TRY(make_map_t(&mc, out16_dev, 2, M, 2 * static_cast<uint64_t>(N), 2 * static_cast<uint64_t>(N), 32));
    EpiBiasF16Wide<true>::Params p{bias_dev, N};
    return launch_gemm_pp<EpiBiasF16Wide<true>>(ma, mb, mc, M, N, K, p, s, sms);
  }
  if (epi == 1) {
    if (N % 32) return fail(B200MDM_EINVAL, "EpiBiasF16Global needs N %% 32 == 0");
    TRY(make_map_t(&mc, out16_dev, 2, M, N, N, 32));
    EpiBiasF16Global::Params p{bias_dev};
    return launch_gemm_pp<EpiBiasF16Global>(ma, mb, mc, M, N, K, p, s, sms);
  }
  return fail(B200MDM_EINVAL, "epi must be 0 (EpiBiasF16Wide<GELU>) or 1 (EpiBiasF16Global)");
}

extern "C" int b200mdm_test_embed(const float* x_dev, const float* w_in_dev, const float* b_in_dev, const float* pe_dev,
                                  void* hres16_dev, int32_t B, int32_t JF, int32_t T, int32_t d, int32_t s_off,
                                  int32_t halves, void* stream) {
  if (!x_dev || !w_in_dev || !b_in_dev || !pe_dev || !hres16_dev || B <= 0 || JF <= 0 || T <= 0 || s_off < 0 ||
      d <= 0 || d % 64 || d * 4 > GEMM_BIAS_BYTES || (halves != 1 && halves != 2))
    return fail(B200MDM_EINVAL, "bad argument (d %% 64 == 0, d <= %d, halves 1 or 2)", GEMM_BIAS_BYTES / 4);
  int sms = 132;
  TRY(test_prologue(&sms));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int S = T + s_off, Kp = (JF + 7) & ~7, MB = B * S;
  StreamScratch scr(s);
  __half *xin16 = nullptr, *w_in3 = nullptr;
  float* pe_bias = nullptr;
  TRY(scr.alloc(&xin16, static_cast<size_t>(MB) * 3 * Kp, true));   // rows s < s_off and the pad columns stay zero
  TRY(scr.alloc(&w_in3, static_cast<size_t>(d) * 3 * Kp, true));
  TRY(scr.alloc(&pe_bias, static_cast<size_t>(S) * d));
  TRY(launch_pack_input(x_dev, xin16, B, JF, T, S, Kp, s_off, s));
  split_weight_kernel<<<d, 128, 0, s>>>(w_in_dev, w_in3, d, JF, Kp);
  CUDA_TRY(cudaGetLastError());
  pe_bias_kernel<<<S, 128, 0, s>>>(pe_bias, pe_dev, b_in_dev, S, d);
  CUDA_TRY(cudaGetLastError());
  CUtensorMap m_xin, m_win, m_res_c, m_res_u;
  TRY(make_map(&m_xin, xin16, MB, 3 * Kp, 3 * Kp, GEMM_BLOCK_M));
  TRY(make_map(&m_win, w_in3, d, 3 * Kp, 3 * Kp, 128));
  TRY(make_map_res(&m_res_c, hres16_dev, MB, d));
  TRY(make_map_res(&m_res_u, static_cast<__half*>(hres16_dev) + (halves == 2 ? static_cast<size_t>(MB) * d * 2 : 0), MB, d));
  return launch_embed_gemm(m_xin, m_win, m_res_c, m_res_u, pe_bias, MB, S, d, Kp, halves, s, sms);
}

// One output-step launch of a test hook, as the step makes it, on scratch memory: g16 = the CFG blend of hres and the
// split output weight; each table a zeroed (index + 1)-row copy, with `row` at `index` of table `table`; the step state
// (done, index, n_steps); and zeroed scratch for the PLMS ring, the partial sums, and the noise, DPM-Solver++ history
// and x_start the caller leaves null.  With `terms`, launch_vb_reduce then reduces the bound's partial sums into it.
struct OutHook {
  const void* hres16;
  const float *scale, *w_out, *b_out;
  int B, JF, T, d, s_off, halves;
  const uint8_t* inpaint_mask;
  const float *inpaint_weight, *inpaint_motion;
  StepArgs a;   // mode, order, clip, const_noise, x_in, noise, x_out (scratch when null), pred
  SchedTable table = TAB_STEP;
  const float* row = nullptr;
  int index = 0, done = 0, n_steps = 0;
  float *x0_hist = nullptr, *vb_elem = nullptr, *terms = nullptr;
  const float* x_start = nullptr;
};
static int run_out_hook(OutHook h, cudaStream_t s) {
  const int B = h.B, JF = h.JF, T = h.T, d = h.d;
  if (!h.hres16 || !h.w_out || !h.b_out || !h.a.x_in || B <= 0 || JF <= 0 || T <= 0 || h.s_off < 0 || d <= 0 || d % 64 ||
      (h.halves != 1 && h.halves != 2) || (h.halves == 2 && !h.scale) ||
      (h.inpaint_mask == nullptr && h.inpaint_weight == nullptr) != (h.inpaint_motion == nullptr))
    return fail(B200MDM_EINVAL, "bad argument");
  int sms = 132;
  TRY(test_prologue(&sms));
  StreamScratch scr(s);
  const int N_out_pad = ((JF + 95) / 96) * 96;
  const size_t n = static_cast<size_t>(B) * JF * T;
  __half *g16 = nullptr, *w_out3 = nullptr;
  TRY(scr.alloc(&g16, static_cast<size_t>(B) * T * 3 * d));
  TRY(scr.alloc(&w_out3, static_cast<size_t>(N_out_pad) * 3 * d, true));
  split_weight_kernel<<<JF, 128, 0, s>>>(h.w_out, w_out3, JF, d, d);
  CUDA_TRY(cudaGetLastError());
  TRY(launch_blend_split(static_cast<const __half*>(h.hres16), g16, h.scale, B, T + h.s_off, T, h.s_off, d, h.halves, nullptr, s));
  CUtensorMap m_g16, m_wout;
  TRY(make_map(&m_g16, g16, static_cast<uint64_t>(B) * T, 3 * d, 3 * d, GEMM_BLOCK_M));
  TRY(make_map(&m_wout, w_out3, N_out_pad, 3 * d, 3 * d, 96));
  EpiOutParams p{};
  p.bias = h.b_out;
  p.inpaint_mask = h.inpaint_mask;
  p.inpaint_weight = h.inpaint_weight;
  p.inpaint_motion = h.inpaint_motion;
  float* tab[N_TABLES];
  for (int t = 0; t < N_TABLES; ++t) TRY(scr.alloc(&tab[t], static_cast<size_t>(h.index + 1) * TAB_STRIDE[t], true));
  if (h.row)
    CUDA_TRY(cudaMemcpyAsync(tab[h.table] + static_cast<size_t>(h.index) * TAB_STRIDE[h.table], h.row,
                             TAB_STRIDE[h.table] * sizeof(float), cudaMemcpyDeviceToDevice, s));
  set_tables(&p, tab);
  StepState* st = nullptr;
  TRY(scr.alloc(&st, 1));
  step_set_kernel<<<1, 1, 0, s>>>(st, h.done, h.index, nullptr, 0, 0, 0, h.n_steps);
  CUDA_TRY(cudaGetLastError());
  p.state = st;
  float* zeros = nullptr;
  TRY(scr.alloc(&zeros, n, true));
  TRY(scr.alloc(&p.eps_ring, PLMS_RING * n, true));
  p.x0_hist = h.x0_hist;
  if (!p.x0_hist) TRY(scr.alloc(&p.x0_hist, DPM_SLOTS * n, true));
  TRY(scr.alloc(&p.vb_part, static_cast<size_t>(VB_TERMS) * B * T * ((JF + 31) / 32), true));
  p.vb_elem = h.vb_elem;
  p.x_start = h.x_start ? h.x_start : zeros;
  if (!h.a.noise) h.a.noise = zeros;
  if (!h.a.x_out) TRY(scr.alloc(&h.a.x_out, n));
  TRY(launch_out_gemm(m_g16, m_wout, B, T, JF, d, h.a, p, s, sms));
  return h.terms ? launch_vb_reduce(h.terms, h.n_steps, p.vb_part, B, T, JF, st, s) : B200MDM_OK;
}

extern "C" int b200mdm_test_out_step(const void* hres16_dev, const float* scale_dev, const float* w_out_dev,
                                     const float* b_out_dev, const float* x_t_dev, const float* noise_dev,
                                     const float* sched_row_dev, int32_t mode, int32_t flags, const uint8_t* inpaint_mask_dev,
                                     const float* inpaint_motion_dev, float* x_out_dev, float* pred_xstart_dev, int32_t B,
                                     int32_t JF, int32_t T, int32_t d, int32_t s_off, int32_t halves, void* stream) {
  if (!x_out_dev || !pred_xstart_dev || mode < B200MDM_MODE_X0 || mode > B200MDM_MODE_DDIM ||
      (mode != B200MDM_MODE_X0 && (!noise_dev || !sched_row_dev)))
    return fail(B200MDM_EINVAL, "bad argument");
  OutHook h{hres16_dev, scale_dev, w_out_dev, b_out_dev, B, JF, T, d, s_off, halves, inpaint_mask_dev, nullptr, inpaint_motion_dev};
  h.a.mode = mode;
  h.a.x_in = x_t_dev;
  h.a.noise = noise_dev;
  h.a.const_noise = flags & B200MDM_FLAG_CONST_NOISE;
  h.a.clip = (flags & B200MDM_FLAG_CLIP_DENOISED) ? 1 : 0;
  h.a.x_out = x_out_dev;
  h.a.pred = pred_xstart_dev;
  h.row = sched_row_dev;
  return run_out_hook(h, static_cast<cudaStream_t>(stream));
}

extern "C" int b200mdm_test_out_dpm(const void* hres16_dev, const float* scale_dev, const float* w_out_dev,
                                    const float* b_out_dev, const float* x_t_dev, const float* dpm_row_dev, int32_t index,
                                    int32_t step, int32_t order, int32_t flags, const uint8_t* inpaint_mask_dev,
                                    const float* inpaint_motion_dev, float* x0_hist_dev, float* x_out_dev, int32_t B,
                                    int32_t JF, int32_t T, int32_t d, int32_t s_off, int32_t halves, void* stream) {
  if (!dpm_row_dev || !x0_hist_dev || !x_out_dev || index < 0 || step < 0 || (order != 1 && order != 2) ||
      (flags & ~B200MDM_FLAG_CLIP_DENOISED))
    return fail(B200MDM_EINVAL, "bad argument");
  OutHook h{hres16_dev, scale_dev, w_out_dev, b_out_dev, B, JF, T, d, s_off, halves, inpaint_mask_dev, nullptr, inpaint_motion_dev};
  h.a.mode = MODE_DPM;
  h.a.order = order;
  h.a.x_in = x_t_dev;
  h.a.clip = (flags & B200MDM_FLAG_CLIP_DENOISED) ? 1 : 0;
  h.a.x_out = x_out_dev;
  h.table = TAB_DPM;
  h.row = dpm_row_dev;
  h.index = index;
  h.done = step;
  h.n_steps = index + 1;
  h.x0_hist = x0_hist_dev;
  return run_out_hook(h, static_cast<cudaStream_t>(stream));
}

extern "C" int b200mdm_test_out_vb(const void* hres16_dev, const float* scale_dev, const float* w_out_dev,
                                   const float* b_out_dev, const float* x_t_dev, const float* x_start_dev, const float* noise_dev,
                                   const float* vb_row_dev, int32_t index, int32_t n_steps, int32_t flags,
                                   const uint8_t* inpaint_mask_dev, const float* inpaint_motion_dev, float* pred_xstart_dev,
                                   float* elem_dev, float* terms_dev, int32_t B, int32_t JF, int32_t T, int32_t d, int32_t s_off,
                                   int32_t halves, void* stream) {
  if (!x_start_dev || !noise_dev || !vb_row_dev || !terms_dev || index < 0 || index >= n_steps ||
      (flags & ~B200MDM_FLAG_CLIP_DENOISED))
    return fail(B200MDM_EINVAL, "bad argument");
  OutHook h{hres16_dev, scale_dev, w_out_dev, b_out_dev, B, JF, T, d, s_off, halves, inpaint_mask_dev, nullptr, inpaint_motion_dev};
  h.a.mode = MODE_VB;
  h.a.x_in = x_t_dev;
  h.a.noise = noise_dev;
  h.a.clip = (flags & B200MDM_FLAG_CLIP_DENOISED) ? 1 : 0;
  h.a.pred = pred_xstart_dev;
  h.table = TAB_VB;
  h.row = vb_row_dev;
  h.index = index;
  h.n_steps = n_steps;
  h.x_start = x_start_dev;
  h.vb_elem = elem_dev;
  h.terms = terms_dev;
  return run_out_hook(h, static_cast<cudaStream_t>(stream));
}

// x0 of the output epilogue with soft inpainting, on the GEMM instantiation of update family `mode` (B200MDM_MODE_X0 /
// DDPM / DDIM: OutStep; 3: OutPlms, 6: OutReverse, 7: OutDpm, 8: OutVb), launched by launch_out_gemm as the step launches
// it.  Every family writes the x0 it formed to pred_xstart; its other outputs and inputs live in zeroed scratch.
extern "C" int b200mdm_test_out_weight(const void* hres16_dev, const float* scale_dev, const float* w_out_dev,
                                       const float* b_out_dev, const float* x_t_dev, int32_t mode, int32_t flags,
                                       const float* weight_dev, const float* motion_dev, float* pred_xstart_dev, int32_t B,
                                       int32_t JF, int32_t T, int32_t d, int32_t s_off, int32_t halves, void* stream) {
  const bool family = mode == MODE_X0 || mode == MODE_DDPM || mode == MODE_DDIM || mode == MODE_PLMS_AB ||
                      mode == MODE_DDIM_REVERSE || mode == MODE_DPM || mode == MODE_VB;
  if (!pred_xstart_dev || !family || (flags & ~B200MDM_FLAG_CLIP_DENOISED)) return fail(B200MDM_EINVAL, "bad argument");
  OutHook h{hres16_dev, scale_dev, w_out_dev, b_out_dev, B, JF, T, d, s_off, halves, nullptr, weight_dev, motion_dev};
  h.a.mode = mode;
  h.a.order = 1;
  h.a.x_in = x_t_dev;
  h.a.clip = (flags & B200MDM_FLAG_CLIP_DENOISED) ? 1 : 0;
  h.a.pred = pred_xstart_dev;
  h.n_steps = 1;
  return run_out_hook(h, static_cast<cudaStream_t>(stream));
}

extern "C" int b200mdm_test_blend_handshake(const void* hres16_dev, const float* scale_dev, void* g16_dev, int32_t B,
                                            int32_t T, int32_t d, int32_t s_off, int32_t halves, int32_t h,
                                            const int64_t* lengths_host, const uint8_t* motion_start_host, void* stream) {
  if (!hres16_dev || !g16_dev || B <= 0 || T <= 0 || s_off < 0 || d <= 0 || d % 64 || (halves != 1 && halves != 2) ||
      (halves == 2 && !scale_dev))
    return fail(B200MDM_EINVAL, "bad argument");
  std::vector<int> desc;
  TRY(handshake_desc(h, B, T, lengths_host, motion_start_host, &desc));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  StreamScratch scr(s);
  int* hs = nullptr;
  if (!desc.empty()) {
    TRY(scr.alloc(&hs, desc.size()));
    CUDA_TRY(cudaMemcpyAsync(hs, desc.data(), desc.size() * sizeof(int), cudaMemcpyHostToDevice, s));
  }
  TRY(launch_blend_split(static_cast<const __half*>(hres16_dev), static_cast<__half*>(g16_dev), scale_dev, B, T + s_off, T,
                         s_off, d, halves, hs, s));
  CUDA_TRY(cudaStreamSynchronize(s));   // `desc` is local
  return B200MDM_OK;
}

extern "C" int b200mdm_test_attention(const void* qkv16_dev, void* out16_dev, const int32_t* kvlen_dev,
                                      int32_t n_samples, int32_t S, int32_t d, int32_t impl, void* stream) {
  if (!qkv16_dev || !out16_dev || !kvlen_dev || n_samples <= 0 || S <= 0) return fail(B200MDM_EINVAL, "bad argument");
  TRY(init_kernel_attrs());
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (impl != 0 && impl != 1) return fail(B200MDM_EINVAL, "impl must be 0 (fp16 output) or 1 ([hi | lo] output)");
  if (S > ATC_MAX_KEYS) return fail(B200MDM_EINVAL, "attention handles at most %d tokens", ATC_MAX_KEYS);
  CUtensorMap mkv;
  TRY(make_attention_kv_map(&mkv, qkv16_dev, n_samples, S, 3 * d));
  return launch_attention_tc(mkv, static_cast<const __half*>(qkv16_dev), static_cast<__half*>(out16_dev), kvlen_dev, n_samples,
                             S, d, d / ATC_DH, s, impl == 1);
}

extern "C" int b200mdm_test_cross_attention(const void* q16_dev, const void* kv16_dev, const unsigned char* mask_dev,
                                            void* out16_dev, int32_t n_samples, int32_t S, int32_t n_tokens, int32_t ld_kv,
                                            void* stream) {
  const int d = 512;
  if (!q16_dev || !kv16_dev || !mask_dev || !out16_dev || n_samples <= 0 || S <= 0 || n_tokens <= 0 || n_tokens > XAL_MAX_MT ||
      ld_kv < 2 * d || ld_kv % 8)
    return fail(B200MDM_EINVAL, "bad argument");
  TRY(init_kernel_attrs());
  return launch_cross_attention(static_cast<const __half*>(q16_dev), static_cast<const __half*>(kv16_dev), mask_dev,
                                static_cast<__half*>(out16_dev), n_samples, S, n_tokens, d, d / 128, ld_kv,
                                static_cast<cudaStream_t>(stream));
}

// QKV projection + attention core of an encoder layer, the two launches the step makes, through a scratch qkv buffer.
extern "C" int b200mdm_test_qkv_attention(const void* h16_dev, int32_t ld, const void* wqkv16_dev, const float* bqkv_dev,
                                          void* out16_dev, const int32_t* kvlen_dev, int32_t n_samples, int32_t S,
                                          void* stream) {
  if (!h16_dev || !wqkv16_dev || !bqkv_dev || !out16_dev || !kvlen_dev || n_samples <= 0 || S <= 0 || S > ATC_MAX_KEYS ||
      ld < 512 || ld % 8)
    return fail(B200MDM_EINVAL, "bad argument");
  int sms = 132;
  TRY(test_prologue(&sms));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int M = n_samples * S;
  __half* qkv = nullptr;
  CUDA_TRY(cudaMallocAsync(reinterpret_cast<void**>(&qkv), static_cast<size_t>(M) * 1536 * sizeof(__half), s));
  CUtensorMap ma, mb, mc, mkv;
  int r = make_map(&ma, h16_dev, M, 512, ld, GEMM_BLOCK_M);
  if (r == B200MDM_OK) r = make_map(&mb, wqkv16_dev, 1536, 512, 512, 128);
  if (r == B200MDM_OK) r = make_map_t(&mc, qkv, 2, M, 1536, 1536, 32);
  if (r == B200MDM_OK) r = launch_gemm_bias<false>(ma, mb, mc, M, 1536, 512, bqkv_dev, s, sms);
  if (r == B200MDM_OK) r = make_attention_kv_map(&mkv, qkv, n_samples, S, 1536);
  if (r == B200MDM_OK)
    r = launch_attention_tc(mkv, qkv, static_cast<__half*>(out16_dev), kvlen_dev, n_samples, S, 512, 4, s);
  CUDA_TRY(cudaFreeAsync(qkv, s));
  return r;
}

extern "C" int b200mdm_test_gemm_resid_ln(const void* a16_dev, const void* w16_dev, const float* bias_dev,
                                          const float* gamma_dev, const float* beta_dev, void* hres16_dev, int32_t M,
                                          int32_t K, void* stream) {
  if (!a16_dev || !w16_dev || !bias_dev || !gamma_dev || !beta_dev || !hres16_dev || M <= 0 || K <= 0 || K % 8)
    return fail(B200MDM_EINVAL, "bad argument");
  int sms = 132;
  TRY(test_prologue(&sms));
  CUtensorMap ma, mb, mh;
  TRY(make_map(&ma, a16_dev, M, K, K, GEMM_BLOCK_M));
  TRY(make_map(&mb, w16_dev, GLN_D, K, K, 256));
  TRY(make_hres_map(&mh, hres16_dev, M));
  return launch_gemm_resid_ln(ma, mb, mh, M, K, bias_dev, gamma_dev, beta_dev, static_cast<cudaStream_t>(stream), sms);
}

extern "C" int b200mdm_test_cross_rows(b200mdm_engine* e, int32_t timestep, float* out_dev, void* stream) {
  if (!e || !out_dev) return fail(B200MDM_EINVAL, "bad argument");
  if (!e->dec_clip) return fail(B200MDM_EINVAL, "cross-attention rows belong to trans_dec engines with a CLIP memory");
  if (!e->finalized || !e->cond_set) return fail(B200MDM_ESTATE, "weights and b200mdm_set_cond_dec first");
  if (timestep < 0 || timestep >= e->cfg.temb_rows) return fail(B200MDM_EINVAL, "timestep outside [0, %d)", e->cfg.temb_rows);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  std::vector<int> t(e->B, timestep);
  CUDA_TRY(cudaMemcpyAsync(e->tvec, t.data(), e->B * sizeof(int), cudaMemcpyHostToDevice, s));
  TRY(launch_cross_rows(e, out_dev, e->tvec, 0, s));
  CUDA_TRY(cudaStreamSynchronize(s));   // `t` is local
  return B200MDM_OK;
}

extern "C" int b200mdm_test_row_bias_ln(void* hres16_dev, const float* c_dev, const float* gamma_dev, const float* beta_dev,
                                        int32_t M, int32_t S, void* stream) {
  if (!hres16_dev || !c_dev || !gamma_dev || !beta_dev || M <= 0 || S <= 0) return fail(B200MDM_EINVAL, "bad argument");
  if ((reinterpret_cast<uintptr_t>(hres16_dev) | reinterpret_cast<uintptr_t>(c_dev) | reinterpret_cast<uintptr_t>(gamma_dev) |
       reinterpret_cast<uintptr_t>(beta_dev)) & 15)
    return fail(B200MDM_EINVAL, "operands must be 16-byte aligned");
  return launch_row_bias_ln(static_cast<__half*>(hres16_dev), c_dev, gamma_dev, beta_dev, M, S, static_cast<cudaStream_t>(stream));
}

#ifdef B200_TRACE
// Instrumented build only: dims <- {CTAs, tile iterations, roles, events} of gemm_resid_ln_cluster's phase stamps; with
// host_out, copies the stamps (uint64 ns, 0 where no launch reached) to it and clears them.  Synchronises the device.
extern "C" int b200mdm_debug_ln_trace(uint64_t* host_out, int32_t* dims) {
  if (!dims) return fail(B200MDM_EINVAL, "bad argument");
  dims[0] = GLN_TRACE_CTAS; dims[1] = GLN_TRACE_ITERS; dims[2] = GLN_TRACE_ROLES; dims[3] = GLN_TRACE_EVENTS;
  if (host_out) {
    CUDA_TRY(cudaDeviceSynchronize());
    CUDA_TRY(cudaMemcpyFromSymbol(host_out, g_gln_trace, sizeof(g_gln_trace)));
    void* dev = nullptr;
    CUDA_TRY(cudaGetSymbolAddress(&dev, g_gln_trace));
    CUDA_TRY(cudaMemset(dev, 0, sizeof(g_gln_trace)));
    CUDA_TRY(cudaDeviceSynchronize());
  }
  return B200MDM_OK;
}
#endif

// The joint terms and the motion shape of a b200mdm_test_*_guidance hook
static int fill_test_joint(const float* x0_dev, const float* x0_out_dev, const float* mean_dev, const float* std_dev,
                           const float* target_dev, const float* weight_dev, int32_t B, int32_t T, int32_t D, float step,
                           int32_t iters, JointGuide* out) {
  if (!x0_dev || !x0_out_dev) return fail(B200MDM_EINVAL, "null argument");
  TRY(fill_joint(mean_dev, std_dev, target_dev, weight_dev, step, iters, out));
  if (D != 263 && D != 251) return fail(B200MDM_EINVAL, "D %d: 263 (HumanML3D) or 251 (KIT)", D);
  if (B < 1 || T < 1 || T > JG_MAX_FRAMES) return fail(B200MDM_EINVAL, "B %d, T %d: B >= 1, 1 <= T <= %d", B, T, JG_MAX_FRAMES);
  return B200MDM_OK;
}

// The b200mdm_test_*_guidance hooks after their checks: the test kernel of the row of `top` (the hook's highest term) on
// descriptor d, with d's lengths and reach rows staged from the host `len` and `rows`, which the hook's return ends, so
// the stream is synchronised when there are any
static int test_guidance(GuideDesc d, unsigned top, const std::vector<int>& len, const std::vector<InterPair>& rows,
                         const float* x0_dev, float* x0_out_dev, float* loss_out_dev, int B, int T, int D, void* stream) {
  const GuideVariant& v = GUIDE_VARIANTS[guide_variant(top)];
  TRY(init_kernel_attrs());
  if (v.clusters) TRY(check_inter_cluster(v.test, d.i.chars, B, T, D));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  int* dlen = nullptr;
  InterPair* dpairs = nullptr;
  if (!len.empty()) {
    CUDA_TRY(cudaMallocAsync(reinterpret_cast<void**>(&dlen), len.size() * sizeof(int), s));
    CUDA_TRY(cudaMemcpyAsync(dlen, len.data(), len.size() * sizeof(int), cudaMemcpyHostToDevice, s));
    d.f.lengths = dlen;
  }
  if (!rows.empty()) {
    CUDA_TRY(cudaMallocAsync(reinterpret_cast<void**>(&dpairs), rows.size() * sizeof(InterPair), s));
    CUDA_TRY(cudaMemcpyAsync(dpairs, rows.data(), rows.size() * sizeof(InterPair), cudaMemcpyHostToDevice, s));
    d.i.pairs = dpairs;
  }
  cudaError_t err = launch_kc(v.test, dim3(B), dim3(JG_THREADS), v.smem(T, ric_dims(D).R), s, v.clusters ? d.i.chars : 0,
                              d, x0_dev, x0_out_dev, loss_out_dev, B, T, D);
  if (err == cudaSuccess) err = cudaGetLastError();
  if (dlen) cudaFreeAsync(dlen, s);
  if (dpairs) cudaFreeAsync(dpairs, s);
  if (err != cudaSuccess) return fail(B200MDM_ECUDA, "%s", cudaGetErrorString(err));
  if (dlen || dpairs) CUDA_TRY(cudaStreamSynchronize(s));
  return B200MDM_OK;
}

extern "C" int b200mdm_test_joint_guidance(const float* x0_dev, const float* mean_dev, const float* std_dev,
                                           const float* target_dev, const float* weight_dev, int32_t B, int32_t T, int32_t D,
                                           float step, int32_t iters, float* x0_out_dev, float* loss_out_dev, void* stream) {
  GuideDesc d{};
  TRY(fill_test_joint(x0_dev, x0_out_dev, mean_dev, std_dev, target_dev, weight_dev, B, T, D, step, iters, &d.j));
  return test_guidance(d, GT_JOINT, {}, {}, x0_dev, x0_out_dev, loss_out_dev, B, T, D, stream);
}

extern "C" int b200mdm_test_foot_guidance(const float* x0_dev, const float* mean_dev, const float* std_dev,
                                          const float* target_dev, const float* weight_dev, const float* contact_dev,
                                          const int64_t* lengths_host, int32_t B, int32_t T, int32_t D, float step,
                                          int32_t iters, float contact_weight, float floor_weight, float floor_height,
                                          float* x0_out_dev, float* loss_out_dev, void* stream) {
  GuideDesc d{};
  std::vector<int> len;
  TRY(fill_test_joint(x0_dev, x0_out_dev, mean_dev, std_dev, target_dev, weight_dev, B, T, D, step, iters, &d.j));
  TRY(fill_foot(contact_weight, floor_weight, floor_height, contact_dev, lengths_host, B, T, &d.f, &len));
  return test_guidance(d, GT_FOOT, len, {}, x0_dev, x0_out_dev, loss_out_dev, B, T, D, stream);
}

extern "C" int b200mdm_test_scene_guidance(const float* x0_dev, const float* mean_dev, const float* std_dev,
                                           const float* target_dev, const float* weight_dev, const float* contact_dev,
                                           const int64_t* lengths_host, int32_t B, int32_t T, int32_t D, float step,
                                           int32_t iters, float contact_weight, float floor_weight, float floor_height,
                                           float obstacle_weight, float obstacle_margin, const b200mdm_grid* sdf,
                                           const b200mdm_grid* terrain, float* x0_out_dev, float* loss_out_dev,
                                           void* stream) {
  GuideDesc d{};
  std::vector<int> len;
  TRY(fill_test_joint(x0_dev, x0_out_dev, mean_dev, std_dev, target_dev, weight_dev, B, T, D, step, iters, &d.j));
  TRY(fill_foot(contact_weight, floor_weight, floor_height, contact_dev, lengths_host, B, T, &d.f, &len));
  TRY(fill_scene(obstacle_weight, obstacle_margin, sdf, terrain, B, &d.f, "", &d.s));
  return test_guidance(d, GT_SCENE, len, {}, x0_dev, x0_out_dev, loss_out_dev, B, T, D, stream);
}

extern "C" int b200mdm_test_interaction_guidance(
    const float* x0_dev, const float* mean_dev, const float* std_dev, const float* target_dev, const float* weight_dev,
    const float* contact_dev, const int64_t* lengths_host, int32_t B, int32_t T, int32_t D, float step, int32_t iters,
    float contact_weight, float floor_weight, float floor_height, float obstacle_weight, float obstacle_margin,
    const b200mdm_grid* sdf, const b200mdm_grid* terrain, int32_t characters, float weight, float margin,
    const float* placement_dev, const int32_t* pairs_host, int32_t n_pairs, const float* reach_host,
    const float* pair_weight_dev, int64_t pair_weight_stride, float* x0_out_dev, float* loss_out_dev, void* stream) {
  GuideDesc d{};
  std::vector<int> len;
  std::vector<InterPair> rows;
  TRY(fill_test_joint(x0_dev, x0_out_dev, mean_dev, std_dev, target_dev, weight_dev, B, T, D, step, iters, &d.j));
  TRY(fill_foot(contact_weight, floor_weight, floor_height, contact_dev, lengths_host, B, T, &d.f, &len));
  TRY(fill_scene(obstacle_weight, obstacle_margin, sdf, terrain, B, &d.f, "", &d.s));
  TRY(fill_inter(characters, weight, margin, placement_dev, pairs_host, n_pairs, reach_host, pair_weight_dev,
                 pair_weight_stride, B, T, D, &d.i, &rows));
  return test_guidance(d, GT_INTER, len, rows, x0_dev, x0_out_dev, loss_out_dev, B, T, D, stream);
}

// ------------------------------------------------------------------------------------------------ post-processing
extern "C" int b200mdm_recover_from_ric(const float* data_dev, int64_t stride_b, int64_t stride_f, int64_t stride_t,
                                        const float* mean_dev, const float* std_dev, float* out_dev, int64_t ostride_b,
                                        int64_t ostride_t, int64_t ostride_c, int32_t batch, int32_t nframes,
                                        int32_t njoints, void* stream) {
  if (!data_dev || !out_dev || batch <= 0 || nframes <= 0 || njoints < 2) return fail(B200MDM_EINVAL, "bad argument");
  if ((mean_dev == nullptr) != (std_dev == nullptr)) return fail(B200MDM_EINVAL, "mean and std come together");
  const size_t smem = static_cast<size_t>(nframes) * 7 * sizeof(float);
  if (smem > 48 * 1024) return fail(B200MDM_ENOTIMPL, "recover_from_ric: %d frames exceed the single-CTA scan", nframes);
  RicArgs a;
  a.x = data_dev; a.xb = stride_b; a.xf = stride_f; a.xt = stride_t;
  a.mean = mean_dev; a.std = std_dev;
  a.out = out_dev; a.ob = ostride_b; a.ot = ostride_t; a.oc = ostride_c;
  a.T = nframes; a.joints = njoints;
  recover_from_ric_kernel<<<batch, 256, smem, static_cast<cudaStream_t>(stream)>>>(a);
  CUDA_TRY(cudaGetLastError());
  return B200MDM_OK;
}

extern "C" int b200mdm_test_target(b200mdm_engine* e, const float* target_dev, const uint8_t* valid_host, int32_t batch,
                                   float* out_dev, void* stream) {
  if (!e || !target_dev || !valid_host || !out_dev || batch <= 0) return fail(B200MDM_EINVAL, "bad argument");
  if (e->cfg.target_encoder == B200MDM_TARGET_NONE) return fail(B200MDM_EINVAL, "this engine has no target encoder");
  if (!e->finalized) return fail(B200MDM_ESTATE, "weights not finalised");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  float* valid = nullptr;
  CUDA_TRY(cudaMallocAsync(reinterpret_cast<void**>(&valid), static_cast<size_t>(batch) * e->cfg.target_joints * sizeof(float), s));
  std::vector<float> staging;
  const int r = encode_target(e, target_dev, valid_host, batch, valid, out_dev, staging, s);
  cudaFreeAsync(valid, s);
  CUDA_TRY(cudaStreamSynchronize(s));   // `staging` is local
  return r;
}
