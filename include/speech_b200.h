/* speech_b200 — C ABI of the H100-native (sm_90a) hot path of awni/speech.
 *
 * Boundary rules (SURVEY.md §8b):
 *   - plain C symbols, raw pointers and sizes, no torch / C++ types in any signature;
 *   - every buffer is caller-owned (PyTorch allocates); the library never allocates device
 *     memory, never synchronises the device, and never throws: each entry point returns an
 *     int status (SB_OK == 0) and enqueues its kernels on the cudaStream_t passed as `stream`
 *     (a void* so that this header needs no CUDA include);
 *   - unless stated otherwise every pointer is a DEVICE pointer;
 *   - re-entrant across streams; one process per GPU.
 *
 * Each entry point cites the reference interface it replaces (paths relative to the
 * reference tree, awni/speech @ a5909a3).
 */
#ifndef SPEECH_B200_H_
#define SPEECH_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SB_OK 0
#define SB_ERR_INVALID 1      /* bad argument */
#define SB_ERR_CUDA 2         /* a CUDA runtime / driver call failed */
#define SB_ERR_UNSUPPORTED 3  /* shape outside what the kernels implement */
#define SB_ERR_WORKSPACE 4    /* caller-provided workspace too small */

/* library / device introspection -------------------------------------------------------- */
int sb_version(void);                 /* 100 * major + minor */
const char* sb_status_string(int status);
int sb_device_info(int* sm_count, int* cc_major, int* cc_minor, size_t* l2_bytes);

/* ---------------------------------------------------------------------------------------
 * CTC loss + gradient.
 * Replaces: functions.ctc.CTCLoss()(acts, labels, act_lens, label_lens)
 *           (libs/warp-ctc pytorch_binding; call site speech/models/ctc_model.py:34-40;
 *            un-vendored dependency cloned by Makefile:4-7).
 *   acts        (B, T, V) float32, batch-first, UN-normalised (softmax is internal)
 *   grads       (B, T, V) float32 out: d(sum_b cost_b)/d acts; may be NULL (costs only)
 *   labels      flat int32 [sum(label_lens)], label_offsets = exclusive prefix sum of label_lens
 *   act_lens    (B) int32 valid frames per utterance (reference passes T for all,
 *               ctc_model.py:43-45); rows >= act_lens[b] get zero gradient
 *   blank       blank class index (reference: V-1, ctc_model.py:18)
 *   costs       (B) float32 out: -log p(labels_b | acts_b); +inf when no alignment exists
 *   workspace   >= sb_ctc_workspace_size(...) bytes
 * ------------------------------------------------------------------------------------- */
int sb_ctc_workspace_size(int B, int T, int V, int max_label_len, size_t* bytes);
int sb_ctc_fwd_bwd(const float* acts, float* grads, const int* labels, const int* label_offsets,
                   const int* label_lens, const int* act_lens, int B, int T, int V, int blank,
                   int max_label_len, float* costs, void* workspace, size_t workspace_bytes,
                   void* stream);

/* Any vocabulary size (csrc/ctc.cu).  The fused kernel above keeps per-class occupancies [4][V] in
 * shared memory next to the lattice rows; shapes where it does not fit (both its staged and its
 * unstaged layouts over 220 KB: V above about 13,000 at T = 247, about 9,900 with 512 to 1023
 * labels) take a compact path inside sb_ctc_fwd_bwd, and every other shape keeps the fused kernel.
 * The compact path reduces each frame, over many CTAs, to Vc = max_label_len + 2 columns (blank,
 * the utterance's distinct label classes, and the log-sum-exp of every other class), runs the same
 * fused kernel on them, and expands the gradient (softmax for the classes left out).  Same costs and
 * gradients up to float32 rounding; max_label_len <= 1023 as above.
 *   sb_ctc_fwd_bwd_compact         the compact path at any shape (same arguments as sb_ctc_fwd_bwd)
 *   sb_ctc_compact_workspace_size  its workspace; sb_ctc_workspace_size returns this size exactly
 *                                  for the shapes where sb_ctc_fwd_bwd takes the compact path */
int sb_ctc_compact_workspace_size(int B, int T, int V, int max_label_len, size_t* bytes);
int sb_ctc_fwd_bwd_compact(const float* acts, float* grads, const int* labels,
                           const int* label_offsets, const int* label_lens, const int* act_lens,
                           int B, int T, int V, int blank, int max_label_len, float* costs,
                           void* workspace, size_t workspace_bytes, void* stream);

/* CTC Viterbi (forced) alignment (csrc/ctc.cu): the single best path through the lattice the
 * loss sums over.  Arguments as sb_ctc_fwd_bwd (raw logits, any V, max_label_len <= 1023).  Every
 * frame is reduced by the compact path's kernels; the log-probability of a kept class at frame t
 * is its compact column minus the frame's full-row log-sum-exp (float32).  The recursion runs in
 * float64 over l' = (blank, y1, blank, ..., yL, blank), S = 2L+1:
 *   d[0][0] = lp(0, blank), d[0][1] = lp(0, y1),
 *   d[t][s] = max(d[t-1][s], d[t-1][s-1], d[t-1][s-2]) + lp(t, l'_s), the s-2 step only where
 *   l'_s is not blank and l'_s != l'_{s-2}; the path ends in S-1 or S-2.
 * Tie rule: on equal scores the predecessor s wins over s-1, and s-1 over s-2; at the end S-1
 * wins over S-2.
 *   path     (B, T) int32 out: the label index j (0-based) frame t is aligned to, -1 for blank,
 *            -2 for frames >= act_lens[b]; all -2 where no alignment exists
 *   scores   (B) float64 out: the path's log-probability; -inf where no alignment exists
 *            (act_lens[b] < L + the number of adjacent repeats: the loss's +inf cost).  An empty
 *            transcript aligns every frame to blank.
 *   workspace >= sb_ctc_viterbi_workspace_size(...) bytes: the compact rows (B*T*(max_label_len+2)
 *            floats), the row log-sum-exps, the column map and 2-bit backpointers (B * T *
 *            ceil((2*max_label_len+1) / 256) * 64 bytes, the count rounded up to 1, 2, 4 or 8).
 * Same argument checks and status codes as sb_ctc_fwd_bwd (path / scores non-NULL too); every
 * SB_ERR_INVALID / SB_ERR_UNSUPPORTED is returned before any launch. */
int sb_ctc_viterbi_workspace_size(int B, int T, int V, int max_label_len, size_t* bytes);
int sb_ctc_viterbi(const float* acts, const int* labels, const int* label_offsets,
                   const int* label_lens, const int* act_lens, int B, int T, int V, int blank,
                   int max_label_len, int* path, double* scores, void* workspace,
                   size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------
 * Dense contraction on wgmma tensor cores:
 *     C[M,N] (f32)  (+)=  A[M,K] (bf16, row-major) * B[N,K]^T (bf16, row-major)  (+ bias[N])
 * Replaces: the cuBLAS/cuDNN GEMMs reached through nn.GRU / nn.Linear
 *           (speech/models/model.py:35-39, 115-133).
 *   lda/ldb/ldc  leading dimensions in ELEMENTS; A and B rows must be 16-byte aligned
 *   flags        SB_GEMM_ACCUMULATE: C += (atomic adds; required when split_k > 1)
 *                SB_GEMM_ROW_REMAP : row m = t*remap_B + b is stored at row b*remap_T + t
 *                                    (time-major -> batch-first), rows with b >= valid_B dropped
 *                SB_GEMM_A_MN      : A is given as [K][M] (lda = elements per K row; M contiguous)
 *                SB_GEMM_B_MN      : B is given as [K][N] (ldb = elements per K row; N contiguous)
 *                                    -- the contraction runs over the ROWS of the matrix, which is
 *                                    how activations [tokens][features] enter a weight gradient
 *                                    (dW = dY^T X): no transposed copies are needed
 * ------------------------------------------------------------------------------------- */
#define SB_GEMM_ACCUMULATE 1
#define SB_GEMM_ROW_REMAP 2
#define SB_GEMM_A_MN 4
#define SB_GEMM_B_MN 8
int sb_gemm_bf16_tn(const void* A, long long lda, const void* B, long long ldb, float* C,
                    long long ldc, const float* bias, int M, int N, int K, int flags, int split_k,
                    int remap_B, int remap_T, int valid_B, void* stream);

/* ---------------------------------------------------------------------------------------
 * GRU recurrence (T-serial part of nn.GRU; the time-batched input projection is sb_gemm_bf16_tn).
 * Replaces: cuDNN RNN behind self.rnn in speech/models/model.py:35-39,73 (gate order r,z,n;
 *           bidirectional) and Transducer.dec_rnn, speech/models/transducer_model.py:23-26,68.
 * Internal layout is TIME-MAJOR with the batch padded to a multiple of 8: row m = t*Bp + b.
 *   gi     [T*Bp][ndir*3H] f32   X W_ih^T + b_ih (forward-direction gates first)
 *   whh    [ndir][3H][H]   bf16  recurrent weights;   bhh [ndir][3H] f32
 *   y      [T*Bp][ndir*H]  f32   h_t (out)
 *   xn     [T*Bp][ndir*H]  bf16  h_t (out; operand of the next projection and of dW_hh)
 *   gates  [T*Bp][ndir][4][H] f32 saved r,z,n,(W_hn h + b_hn) for backward (out; may be NULL)
 *   workspace  >= sb_gru_fwd_workspace_size bytes, 1024-byte aligned: per-chunk ready counters
 *          and the double-buffered exchange tiles of h_t (zeroed by the call itself)
 * Constraints: H % 16 == 0, Bp % 8 == 0, Bp <= 128, and either ndir*H/16 <= number of SMs
 *   (W_hh slices resident in shared memory) or, for wider layers, H % U == 0 and
 *   ndir*H/U <= number of SMs for U = 16 or 32 (the wide kernel: U units per CTA, W_hh partly streamed
 *   from L2 every step).  Ceiling: ndir*H <= 32 * SMs (2112 bidirectional, 4224 unidirectional
 *   on a 132-SM H100 SXM).
 * ------------------------------------------------------------------------------------- */
int sb_gru_fwd_workspace_size(int Bp, int H, int ndir, size_t* bytes);
int sb_gru_fwd(const float* gi, const void* whh_bf16, const float* bhh, float* y, void* xn_bf16,
               float* gates, void* workspace, size_t workspace_bytes, int T, int Bp, int H,
               int ndir, void* stream);

/* The forward recurrence resumed from a given state, for streaming: T new frames continue from
 * h_{-1} = h0 instead of 0.  One direction only (SB_ERR_UNSUPPORTED for ndir = 2).
 *   h0     [Bp][H] f32 and h0_bf16 [Bp][H] bf16: the state and the bf16 operand the first step's
 *          W_hh product reads (the fp32 y and the bf16 xn of the previous call's last frame)
 *   gi     [T*Bp][3H] f32 as for sb_gru_fwd
 *   y, xn  [(T+1)*Bp][H]: frame 0 receives h0 / h0_bf16 (copied unless they already are frame 0),
 *          frames 1..T are h_0 .. h_{T-1}
 *   gates  [(T+1)*Bp][4][H] or NULL; frame 0 is left as it was
 * Same workspace, constraints and kernel selection as sb_gru_fwd at (Bp, H, 1), and the same
 * arithmetic: running frames [0, T1) with sb_gru_fwd and then [T1, T) from its last state gives
 * y and xn bit-identical to one sb_gru_fwd over [0, T). */
int sb_gru_fwd_h0(const float* gi, const void* whh_bf16, const float* bhh, const float* h0,
                  const void* h0_bf16, float* y, void* xn_bf16, float* gates, void* workspace,
                  size_t workspace_bytes, int T, int Bp, int H, int ndir, void* stream);

/* "Parity mode" forward recurrence: the same time loop in plain fp32 on CUDA cores (fp32 weights
 * [ndir][3H][H], fp32 state, no bf16 rounding anywhere), csrc/gru_f32.cu.  It exists to measure
 * the bf16 tensor-core path against (SURVEY.md section 7), not to be fast.
 *   barrier: ndir u32 words (zeroed by the call).  Constraints: H % 4 == 0, Bp <= 128,
 *   H/8 <= number of SMs. */
int sb_gru_fwd_f32(const float* gi, const float* whh_f32, const float* bhh, float* y,
                   unsigned int* barrier, int T, int Bp, int H, int ndir, void* stream);

/* Backward through the recurrence.
 *   dy     [T*Bp][ndir*H] f32  gradient w.r.t. y
 *   whh    [ndir][3H][H] bf16  recurrent weights as stored (the same operand sb_gru_fwd takes;
 *          the kernel transposes its slice while staging it into shared memory)
 *   dgi    [T*Bp][ndir*3H] bf16 (out) gradient w.r.t. gi  -> dX = dgi * W_ih, dW_ih, dW_hh (r,z)
 *   dghn   [T*Bp][ndir*H] bf16 (out) r * dn_pre            -> dW_hh (n rows)
 *          (the weight gradients contract these token-major operands directly with
 *           SB_GEMM_A_MN | SB_GEMM_B_MN; no transposed copies exist)
 *   dbih, dbhh [ndir*3H] f32 accumulated (+=)
 *   workspace  >= sb_gru_bwd_workspace_size bytes, 1024-byte aligned (zeroed by the call itself;
 *          at widths that run the wide kernel it also holds W_hh^T, ndir*3H*H bf16)
 * Constraints: those of sb_gru_fwd.
 */
int sb_gru_bwd_workspace_size(int Bp, int H, int ndir, size_t* bytes);
int sb_gru_bwd(const float* dy, const float* y, const float* gates, const void* whh_bf16,
               void* dgi_bf16, void* dghn_bf16, float* dbih, float* dbhh, void* workspace,
               size_t workspace_bytes, int T, int Bp, int H, int ndir, void* stream);

/* Width Hp >= H at which sb_gru_fwd / sb_gru_bwd run a layer of H hidden units: H rounded up to
 * a multiple of 16, if both calls accept that width with the resident kernels: the constraints
 * above, the shared-memory ring of each pass and the co-residency of its grid on the current
 * device.  Otherwise the width of the wide kernels: H rounded up to a multiple of U, U = 16 or 32
 * the smallest whose grid of ndir*Hp/U CTAs fits on the SMs, so Hp - H < U, provided both wide
 * passes fit in shared memory and are co-resident.  SB_ERR_UNSUPPORTED past the ceiling above
 * (the answer needs a CUDA device).  The caller pads the layer with Hp - H zero units per direction (zero W_ih / W_hh rows, W_hh
 * columns and biases; zero W_ih columns of the next layer): they stay exactly 0 for all t. */
int sb_gru_plan(int Bp, int H, int ndir, int* Hp);

/* Per-utterance time alignment of a block of columns of a time-major [T*Bp][ld] matrix (row
 * m = t*Bp + b), for the exact-lengths mode of the GRU stack (csrc/lengths.cu):
 *   right != 0: row (t, b) moves to (t + T - len_b, b)  (each utterance ends at frame T-1)
 *   right == 0: row (t, b) moves to (t - T + len_b, b)  (the inverse: back to frame 0)
 * Destination rows with no source row are zero-filled.  With right-aligned operands the reverse
 * direction of sb_gru_fwd / sb_gru_bwd processes each utterance's real frames first and its
 * padding last, so its real frames are those of the unpadded utterance.
 *   src, dst    first element of the column block; ld_src / ld_dst in elements; out of place only
 *   lens        (Bp) int32 valid frames per row b (device; clamped to [0, T]; give T for padding
 *               rows of the batch)
 *   cols        columns in the block;  elem_bytes 2 (bf16) or 4 (f32) */
int sb_time_align(const void* src, long long ld_src, void* dst, long long ld_dst, const int* lens,
                  int T, int Bp, int cols, int elem_bytes, int right, void* stream);

/* Lookahead (row) convolution above a unidirectional GRU stack (Deep Speech 2, Amodei et al.
 * 2016, section 3.5), csrc/lookahead.cu:  r[t, b, d] = sum_{j=0..tau} W[j][d] * h[t + j, b, d].
 * Replaces: nothing in the reference; the model's nn.Conv1d(H, H, tau + 1, groups=H, bias=False)
 * applied to the right-zero-padded top layer output.
 *   h      [T*Bp][Hp] f32   top layer output y as sb_gru_fwd writes it (row t*Bp + b)
 *   w      [tau+1][Hp] f32  taps, tap-major, zero for padded units
 *   lens   (Bp) int32 valid frames per row (device; clamped to [0, T]) or NULL: T for every row
 *   r      [T*Bp][Hp] f32 (out, may be NULL), rb [T*Bp][Hp] bf16 (out, may be NULL; not both)
 * Arithmetic (streaming relies on it to reproduce the offline pass bit for bit):
 *   - r[t, b, d] for t < len_b is one fp32 FMA chain from 0 over j = 0..tau in ascending order;
 *   - a term with t + j >= len_b is skipped, not multiplied by zero;
 *   - r = 0 at t >= len_b, and rb is the round-to-nearest-even bf16 of r.
 * So r at frame t depends only on h[t .. min(t + tau, len_b - 1)] and on whether len_b cuts the
 * window: a frame whose whole window lies below len_b has the same bits for any larger len_b.
 *
 * sb_lookahead_bwd, from dr = dL/dr [T*Bp][Hp] f32 (read once per tile, like h):
 *   dh [T*Bp][Hp] f32 (out): dh[t] = sum_j W[j] dr[t - j] over t - j >= 0 (ascending j);
 *                            dh = 0 at t >= len_b
 *   dw [tau+1][Hp] f32 (out, overwritten): dW[j][d] = sum over rows b < Bp and t + j < len_b of
 *                            dr[t, b, d] h[t + j, b, d], reduced deterministically: fixed
 *                            per-CTA partials in the workspace, then a reduction of fixed shape,
 *                            so two calls give identical bits
 *   workspace  >= sb_lookahead_bwd_workspace_size(T, Bp, Hp, tau) bytes, 4-byte aligned
 * Refusals, before any CUDA call: SB_ERR_INVALID for a NULL required pointer, T < 1, or both
 * forward outputs NULL; SB_ERR_UNSUPPORTED for tau outside [1, 32], Bp not a multiple of 8 in
 * [8, 128], or Hp not a positive multiple of 8; SB_ERR_WORKSPACE for a short workspace. */
int sb_lookahead_fwd(const float* h, const float* w, const int* lens, float* r, void* rb_bf16,
                     int T, int Bp, int Hp, int tau, void* stream);
int sb_lookahead_bwd_workspace_size(int T, int Bp, int Hp, int tau, size_t* bytes);
int sb_lookahead_bwd(const float* dr, const float* h, const float* w, const int* lens, float* dh,
                     float* dw, void* workspace, size_t workspace_bytes, int T, int Bp, int Hp,
                     int tau, void* stream);

/* ---------------------------------------------------------------------------------------
 * CTC prefix beam search, one CTA per utterance.
 * Replaces: speech.models.ctc_decoder.decode(probs, beam_size, blank)
 *           (speech/models/ctc_decoder.py:38-113; called per utterance by CTC.infer,
 *            speech/models/ctc_model.py:55-60).
 *   logp        (B, T, S) float32 LOG-probabilities (the reference takes np.log of its input
 *               first, ctc_decoder.py:52)
 *   lens        (B) int32 frames to decode per utterance (<= T)
 *   out_labels  (B, T) int32, out_lens (B) int32: best prefix of each utterance
 *   out_scores  (B) float64: negative log-likelihood of that prefix (ctc_decoder.py:112-113)
 * beam_size <= 32.  Lattice arithmetic is float64, ties are broken like the reference's
 * stable sort over dict insertion order.
 * Any S: where the K*S + K candidates of a frame do not fit in shared memory (K*(S+1)*13 bytes over
 * 200 KB), sb_ctc_prefix_beam runs the shortlist search; every other shape keeps the full scan.
 *   sb_ctc_prefix_beam_shortlist  the shortlist search at any shape (same arguments): a pre-pass
 *       writes each frame's 2K+1 most probable non-blank symbols, and each entry scores only those,
 *       its own last symbol and its stay candidate; a per-frame bound check (csrc/decode.cu) falls
 *       back to a full scan of the frame where it cannot prove the selection complete.  Hypotheses,
 *       lengths and float64 scores are bit-identical to the full scan.
 * The workspace size has no S argument, so it always includes the shortlists, B*T*(2K+1) ints.
 * ------------------------------------------------------------------------------------- */
int sb_ctc_prefix_beam_workspace_size(int B, int T, int beam_size, size_t* bytes);
int sb_ctc_prefix_beam(const float* logp, const int* lens, int B, int T, int S, int beam_size,
                       int blank, int* out_labels, int* out_lens, double* out_scores,
                       void* workspace, size_t workspace_bytes, void* stream);
int sb_ctc_prefix_beam_shortlist(const float* logp, const int* lens, int B, int T, int S,
                                 int beam_size, int blank, int* out_labels, int* out_lens,
                                 double* out_scores, void* workspace, size_t workspace_bytes,
                                 void* stream);

/* ---------------------------------------------------------------------------------------
 * CTC prefix beam search with shallow fusion of a token-level backoff n-gram LM.
 * The LM is over the model's own output classes (the blank is never an LM token), orders 1..10.
 * Its device tables (built by speech_b200.lm.NGramLM) are one open-addressed map, linear probing,
 * slot h = ((key * 0x9E3779B97F4A7C15) mod 2^64 >> 32) & (cap - 1), with two kinds of key:
 *   (c << 32) | ((t + 1) << 1) | 0  -> context node of "context c preceded by token t"
 *   (c << 32) | ((t + 1) << 1) | 1  -> index into logp of the n-gram "context c, then token t"
 * Context nodes form a trie over contexts read most recent token first; node 0 is the empty
 * context.  Every context of a stored n-gram has a node, so a walk that stops at depth m proves
 * that no longer context of that entry holds an n-gram.
 * lm(s | h), h the last order-1 symbols of the prefix preceded by <s> where it is shorter, is the
 * ARPA backoff value in natural log: acc = 0, then acc += bow[h'] for each context h' of h from
 * the longest down while (h', s) is not stored, then acc += logp[(h', s)].
 * Fusion: extending beam entry i by symbol s uses q = p_s + (lm_weight * lm(s | ctx_i) +
 * insertion_bonus) for p_s in every term of that extension (float64, in that order).  Blank terms
 * and the repeated symbol that keeps the prefix use p_s.  The returned score is
 * -lse(p_b, p_nb) of the best prefix: acoustic + lm_weight * LM + insertion_bonus * length.
 * With lm_weight = insertion_bonus = 0 the results equal sb_ctc_prefix_beam's bit for bit.
 * ------------------------------------------------------------------------------------- */
#define SB_LM_MAX_ORDER 10
typedef struct SbNgramLm {
  const unsigned long long* keys;  /* [cap] map keys, 0 = empty slot (device) */
  const int* vals;                 /* [cap] context node or logp index (device) */
  const double* logp;              /* [n-grams] natural-log probability (device) */
  const double* bow;               /* [context nodes] natural-log backoff weight, 0 where the
                                      ARPA model stores none (device) */
  const int* tok;                  /* [num_classes] LM token of each class; a class the LM does
                                      not know maps to the token of <unk>; every class but the
                                      blank maps to a token with a unigram (device) */
  int cap;                         /* power of two, at least twice the number of keys */
  int order;                       /* 1 .. SB_LM_MAX_ORDER */
  int num_classes;                 /* classes tok covers; must be >= S */
  int bos;                         /* token of <s> */
  int blank;                       /* the class that is not an LM token; must equal the search's */
  double lm_upper;                 /* >= every lm(s | h): the largest logp plus, per order, the
                                      largest positive bow of that order */
  double lm_abs;                   /* >= |every partial sum of a lookup|: the largest |logp| plus,
                                      per order, the largest |bow| of that order */
} SbNgramLm;

/*   sb_ctc_prefix_beam_lm_workspace_size  bytes for (B, T, beam_size, order)
 *   sb_ctc_prefix_beam_lm                 sb_ctc_prefix_beam's arguments and route choice, plus
 *                                         the LM (host struct of device pointers) and the weights
 *   sb_ctc_prefix_beam_lm_shortlist       the shortlist search at any shape (same arguments);
 *                                         bit-identical to the full scan with the same LM
 * SB_ERR_INVALID for lm_weight < 0, a non-finite weight or bound, lm->num_classes < S, or
 * lm->blank != blank;
 * SB_ERR_UNSUPPORTED for order > SB_LM_MAX_ORDER or beam_size > 32. */
int sb_ctc_prefix_beam_lm_workspace_size(int B, int T, int beam_size, int order, size_t* bytes);
int sb_ctc_prefix_beam_lm(const float* logp, const int* lens, int B, int T, int S, int beam_size,
                          int blank, const SbNgramLm* lm, double lm_weight,
                          double insertion_bonus, int* out_labels, int* out_lens,
                          double* out_scores, void* workspace, size_t workspace_bytes,
                          void* stream);
int sb_ctc_prefix_beam_lm_shortlist(const float* logp, const int* lens, int B, int T, int S,
                                    int beam_size, int blank, const SbNgramLm* lm,
                                    double lm_weight, double insertion_bonus, int* out_labels,
                                    int* out_lens, double* out_scores, void* workspace,
                                    size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------
 * Resumable CTC prefix beam search, for streaming: B independent streams whose beams live in a
 * device state buffer between calls, so that each call advances a stream by the frames that have
 * arrived.  Frames [0, T) searched in any chunking give labels, lengths and float64 scores
 * bit-identical to sb_ctc_prefix_beam[_lm] over [0, T): every call runs the same per-frame code,
 * the tie and route rules are those of the offline search, and trie nodes are numbered by the
 * absolute frame (1 + t*K + r), as one pass over the whole utterance numbers them.
 *   sb_ctc_stream_state_size   bytes of the state of B streams of at most max_frames frames each
 *       (order: 0 without an LM, else the LM's).  Layout: per stream, the beam (p_b, p_nb, trie
 *       node, last symbol and parent node of each of <= K entries), the entries' LM contexts, the
 *       frames consumed and an overflow flag; then the tries of the B streams, max_frames*K + 1
 *       nodes each.
 *   sb_ctc_stream_reset        streams [first, first + count) back to the empty prefix at frame 0;
 *       the other streams are untouched.  Every stream must be reset before its first step.
 *   sb_ctc_stream_step[_lm]    logp (B, T, S) float32 log-probabilities of the new frames, n (B)
 *       int32 on the device: stream b advances by min(n[b], T) frames (0 leaves it as it was).  The
 *       route is chosen as sb_ctc_prefix_beam chooses it; the _shortlist forms force the shortlist
 *       search.  workspace >= sb_ctc_stream_workspace_size(B, T, beam_size): the shortlists.  The
 *       LM arguments are those of sb_ctc_prefix_beam_lm; a state must be stepped with or without
 *       an LM throughout, from its reset on.  A stream asked to pass max_frames is advanced only
 *       to max_frames and its overflow flag is set (the caller, who knows every stream's frame
 *       count, should refuse such a step instead).
 *   sb_ctc_stream_best         each stream's best prefix so far: out_labels (B, max_frames) int32,
 *       out_lens (B), out_scores (B) float64 -lse(p_b, p_nb) of beam entry 0, out_overflow (B).
 * B, max_frames and beam_size must be the same in every call on one state.
 * SB_ERR_INVALID for a null pointer, B, max_frames, T or beam_size <= 0, blank outside [0, S), and
 * every LM argument sb_ctc_prefix_beam_lm refuses; SB_ERR_UNSUPPORTED for beam_size > 32 or
 * order > SB_LM_MAX_ORDER; SB_ERR_WORKSPACE for a short workspace.  All before any CUDA call.
 * ------------------------------------------------------------------------------------- */
int sb_ctc_stream_state_size(int B, int max_frames, int beam_size, int order, size_t* bytes);
int sb_ctc_stream_workspace_size(int B, int T, int beam_size, size_t* bytes);
int sb_ctc_stream_reset(void* state, int B, int max_frames, int beam_size, int first, int count,
                        void* stream);
int sb_ctc_stream_step(const float* logp, const int* n, int B, int T, int S, int beam_size,
                       int blank, int max_frames, void* state, void* workspace,
                       size_t workspace_bytes, void* stream);
int sb_ctc_stream_step_shortlist(const float* logp, const int* n, int B, int T, int S,
                                 int beam_size, int blank, int max_frames, void* state,
                                 void* workspace, size_t workspace_bytes, void* stream);
int sb_ctc_stream_step_lm(const float* logp, const int* n, int B, int T, int S, int beam_size,
                          int blank, const SbNgramLm* lm, double lm_weight,
                          double insertion_bonus, int max_frames, void* state, void* workspace,
                          size_t workspace_bytes, void* stream);
int sb_ctc_stream_step_lm_shortlist(const float* logp, const int* n, int B, int T, int S,
                                    int beam_size, int blank, const SbNgramLm* lm,
                                    double lm_weight, double insertion_bonus, int max_frames,
                                    void* state, void* workspace, size_t workspace_bytes,
                                    void* stream);
int sb_ctc_stream_best(const void* state, int B, int max_frames, int beam_size, int* out_labels,
                       int* out_lens, double* out_scores, int* out_overflow, void* stream);
/*   sb_ctc_stream_nbest        every stored beam entry of every stream, the N-best of two-pass
 *       decoding: out_count (B) int32 the n_b <= K entries of stream b's beam; entry i of stream b
 *       has its labels at out_labels[(b*K + i) * max_frames ..] (B, K, max_frames) int32, its
 *       length at out_lens[b*K + i] (B, K) int32 and c_i = lse(p_b, p_nb), the log-probability
 *       itself (not negated), at out_scores[b*K + i] (B, K) float64.  Slots i >= n_b get length -1
 *       and score -inf.  The order is the order the search stores: each frame's beam is taken as
 *       the first K candidates by (score desc, first-touch rank asc), so entry 0 is the best
 *       (sb_ctc_stream_best's result, whose score is -c_0), and the others follow by score, ties
 *       in the search's first-touch order.  Changes no state.  Serves states stepped without an
 *       LM: with a word LM the stored order is not the end-of-utterance order (that rule is
 *       sb_ctc_stream_best_wordlm's); with a character LM c_i holds the fused scores.
 *       The offline N-best is this same path: sb_ctc_stream_reset, one sb_ctc_stream_step over all
 *       frames with n = each utterance's frames, then sb_ctc_stream_nbest; by the guarantee above
 *       its entry 0 is sb_ctc_prefix_beam's result bit for bit.
 *       SB_ERR_INVALID / SB_ERR_UNSUPPORTED as sb_ctc_stream_best, before any CUDA call. */
int sb_ctc_stream_nbest(const void* state, int B, int max_frames, int beam_size, int* out_labels,
                        int* out_lens, double* out_scores, int* out_count, void* stream);
/* Developer counter: frames the LM-fused shortlist search (character or word LM) rescanned in
 * full, over every call since the last query (synchronous: waits for the device); resets it. */
int sb_debug_ctc_lm_rescans(unsigned long long* frames);

/* ---------------------------------------------------------------------------------------
 * CTC prefix beam search with a word n-gram LM (Hannun et al. 2014, arXiv:1408.2873): the LM
 * scores a word when the delimiter class that ends it (the space of a character model) is
 * emitted, and a lexicon tracks the partial word.
 * A prefix splits at every delimiter into completed words w_1..w_n and a partial word (the
 * classes after the last delimiter).  Each beam entry carries its lexicon node (0 = the root,
 * the empty partial word; -1 = the partial word has left the lexicon) and its last order-1
 * completed words' tokens (most recent first, <s> before the first).  Extending entry i by class
 * s != blank replaces p_s by q in every term of that extension, as the character LM does:
 *   s the delimiter, partial word empty:      q = p_s (leading and repeated delimiters are free);
 *   s the delimiter, partial word non-empty:  q = p_s + ((lm_weight * lm(w | ctx_i) +
 *       insertion_bonus) + g_i) in float64, in that order.  w is the word at i's node, or <unk>
 *       where the node is not a word or is -1; g_i = oov_penalty where the node is >= 1 and not a
 *       word (an OOV word not charged yet), else 0.  The new entry's history is (w, older..) and
 *       its node the root;
 *   s any other class:  q = p_s + oov_penalty where i's node is >= 0 and has no child s (the new
 *       node is -1: the word leaves the lexicon); otherwise q = p_s and the node becomes that
 *       child, or stays -1.
 * Blank terms and the repeated symbol that keeps the prefix use p_s.  lm(w | ctx) is the backoff
 * lookup of the word n-gram, as sb_ctc_prefix_beam_lm's over tokens.
 * End of utterance: each final entry scores final_i = lse(p_b, p_nb) + (e_i + lm_weight *
 * lm(</s> | ctx'_i)), e_i the delimiter term above (0 for an empty partial word) and ctx'_i the
 * history with the trailing word, if there is one.  The result is the entry with the largest
 * final_i (ties: the lowest beam index) and its score -final_i: acoustic + lm_weight * (word LM
 * with </s>) + insertion_bonus * words + oov_penalty * OOV words.
 * oov_penalty <= 0: 0 is an open-vocabulary search scoring OOV words as <unk>, -inf a closed
 * vocabulary.  With lm_weight = insertion_bonus = oov_penalty = 0 the results equal
 * sb_ctc_prefix_beam's bit for bit.
 * Shortlist route: each entry also scores the delimiter on every frame (as it scores its last
 * symbol), and every other class has q <= p_s, so the LM-less bound check applies unchanged.
 * Tables (built by speech_b200.lm.WordLM): the word n-gram in SbNgramLm's layout over tokens
 * w -> w (0..W-1), <s> W, </s> W + 1, <unk> W + 2, with tok the identity over those W + 3 tokens
 * and blank -1; the lexicon as a second map of the same hash and key layout,
 *   (node << 32) | ((class + 1) << 1) | 0  -> child node,
 * and lex_word[node], the word token ending at each node (-1 for none).
 * ------------------------------------------------------------------------------------- */
typedef struct SbWordLm {
  SbNgramLm ngram;                 /* the word n-gram (orders 1 .. SB_LM_MAX_ORDER) */
  const unsigned long long* lex_keys;  /* [lex_cap] lexicon map keys, 0 = empty (device) */
  const int* lex_vals;             /* [lex_cap] child node (device) */
  const int* lex_word;             /* [lexicon nodes] word token of each node or -1 (device) */
  int lex_cap;                     /* power of two, at least twice the number of lexicon edges */
  int num_words;                   /* W >= 1 */
  int has_unk;                     /* the n-gram has a <unk> unigram; else oov_penalty = -inf */
  int num_classes;                 /* classes the lexicon is spelled in; must be >= S */
  int blank;                       /* must equal the search's */
  int delimiter;                   /* the class that ends a word; in [0, S), not the blank */
} SbWordLm;

/*   sb_ctc_prefix_beam_wordlm            sb_ctc_prefix_beam's arguments, route choice and
 *                                        workspace, plus the LM and its three weights
 *   sb_ctc_prefix_beam_wordlm_shortlist  the shortlist search at any shape (same arguments)
 *   sb_ctc_stream_step_wordlm[_shortlist]  sb_ctc_stream_step's arguments plus the LM and weights;
 *       the state is sized with the LM's order and must be stepped with this LM from its reset on
 *   sb_ctc_stream_best_wordlm            sb_ctc_stream_best with the end-of-utterance rule applied
 *                                        to each stored beam (the same LM and weights)
 * SB_ERR_INVALID for a null table, lm_weight < 0 or not finite, insertion_bonus not finite,
 * oov_penalty > 0 or NaN, oov_penalty != -inf without <unk>, lm->num_classes < S, lm->blank !=
 * blank, a delimiter outside [0, S) or equal to the blank, or order < 1;
 * SB_ERR_UNSUPPORTED for order > SB_LM_MAX_ORDER or beam_size > 32.  All before any CUDA call. */
int sb_ctc_prefix_beam_wordlm(const float* logp, const int* lens, int B, int T, int S,
                              int beam_size, int blank, const SbWordLm* lm, double lm_weight,
                              double insertion_bonus, double oov_penalty, int* out_labels,
                              int* out_lens, double* out_scores, void* workspace,
                              size_t workspace_bytes, void* stream);
int sb_ctc_prefix_beam_wordlm_shortlist(const float* logp, const int* lens, int B, int T, int S,
                                        int beam_size, int blank, const SbWordLm* lm,
                                        double lm_weight, double insertion_bonus,
                                        double oov_penalty, int* out_labels, int* out_lens,
                                        double* out_scores, void* workspace,
                                        size_t workspace_bytes, void* stream);
int sb_ctc_stream_step_wordlm(const float* logp, const int* n, int B, int T, int S, int beam_size,
                              int blank, const SbWordLm* lm, double lm_weight,
                              double insertion_bonus, double oov_penalty, int max_frames,
                              void* state, void* workspace, size_t workspace_bytes, void* stream);
int sb_ctc_stream_step_wordlm_shortlist(const float* logp, const int* n, int B, int T, int S,
                                        int beam_size, int blank, const SbWordLm* lm,
                                        double lm_weight, double insertion_bonus,
                                        double oov_penalty, int max_frames, void* state,
                                        void* workspace, size_t workspace_bytes, void* stream);
int sb_ctc_stream_best_wordlm(const void* state, int B, int max_frames, int beam_size,
                              const SbWordLm* lm, double lm_weight, double insertion_bonus,
                              double oov_penalty, int* out_labels, int* out_lens,
                              double* out_scores, int* out_overflow, void* stream);

/* ---------------------------------------------------------------------------------------
 * Conv2d(+ReLU) front-end as im2col + sb_gemm_bf16_tn.
 * Replaces: the cuDNN convolutions behind nn.Conv2d in Model.encode
 *           (speech/models/model.py:19-29,60-71; valid conv, kernel (kh,kw), stride s both dims).
 * Activations are pixel-major channels-last f32 P[(b*To+t)*Fo+f][c] (= the GEMM's C matrix, ReLU
 * applied on read); the im2col matrix is A[m][(i*kw+j)*Ci+ci] bf16 with K padded to Kp.
 *   sb_conv_im2col       src P (or the (B,T,F) input with Ci=1) -> A
 *   sb_conv_relu_to_bct  C of the last layer -> (B, To, Co*Fo) f32 with ReLU (model.py:66-71)
 *   sb_conv_dtop         dY (B,To,Co*Fo) * (C>0) -> dC bf16 [M][Co]; db[c] += column sums
 *   sb_conv_col2im_relu  dA f32 [M][ldA] -> dC of the layer below (gather, masked by Pprev>0)
 * ------------------------------------------------------------------------------------- */
/* `mask_u8` (may be NULL): dropout keep-bytes (1 keep, 0 drop) of the activations involved, same
 * pixel-major channels-last layout as those activations; kept values are multiplied by `mscale`
 * = 1/(1-p) (nn.Dropout after ReLU, model.py:25-26). */
int sb_conv_im2col(const float* src, const void* mask_u8, float mscale, void* dst_bf16, int B,
                   int Ti, int Fi, int Ci, int kh, int kw, int stride, int Kp, int relu,
                   void* stream);
int sb_conv_relu_to_bct(const float* C, const void* mask_u8, float mscale, float* out, int B,
                        int To, int Fo, int Co, void* stream);
int sb_conv_dtop(const float* dY, const float* C, const void* mask_u8, float mscale,
                 void* dC_bf16, float* db, int B, int To, int Fo, int Co, void* stream);
int sb_conv_col2im_relu(const float* dA, long long ldA, const float* Pprev,
                        const void* maskprev_u8, float mscale, void* dCprev_bf16, float* db, int B,
                        int Ti, int Fi, int Ci, int kh, int kw, int stride, void* stream);
/* Direct convolution of a layer past the first (no patch matrix): the footprint of each output
 * tile is staged in shared memory as im2col stages A (ReLU, dropout, bf16), so the operands equal
 * the im2col path's.  Wp is the [Co][ldw] bf16 weight matrix of the im2col path (K order
 * (i, j, ci)).  sb_conv_direct_ok: 1 when all three kernels take the layer (Ci, Co multiples of 8,
 * Co <= 32, resident weights and footprint within shared memory), else 0 (use im2col).
 *   sb_conv_fwd_direct    P (ReLU on read) -> C [M][Co] f32 = conv + bias
 *   sb_conv_dgrad_direct  dC bf16 [M][Co] -> dC of the layer below, as sb_conv_col2im_relu
 *   sb_conv_wgrad_direct  dWT [K][Co] f32 += sum over pixels of act * dC (fp32 atomics) */
int sb_conv_direct_ok(int Fi, int Ci, int Co, int kh, int kw, int stride);
int sb_conv_fwd_direct(const float* P, const void* mask_u8, float mscale, const void* Wp_bf16,
                       int ldw, const float* bias, float* C, int B, int Ti, int Fi, int Ci, int Co,
                       int kh, int kw, int stride, void* stream);
int sb_conv_dgrad_direct(const void* dC_bf16, const void* Wp_bf16, int ldw, const float* Pprev,
                         const void* maskprev_u8, float mscale, void* dCprev_bf16, float* db,
                         int B, int Ti, int Fi, int Ci, int Co, int kh, int kw, int stride,
                         void* stream);
int sb_conv_wgrad_direct(const float* P, const void* mask_u8, float mscale, const void* dC_bf16,
                         float* dWT, int B, int Ti, int Fi, int Ci, int Co, int kh, int kw,
                         int stride, void* stream);

/* ---------------------------------------------------------------------------------------
 * Tail of the training step over flat fp32 buffers.
 * Replaces: nn.utils.clip_grad_norm(model.parameters(), 200) + torch.optim.SGD.step()
 *           (train.py:32-35, 95-97).
 *   sb_sumsq          out[0] = sum(g^2), one pass over the gradient; per-CTA partials combined in
 *                     a fixed order (bit-reproducible: data-parallel replicas stay identical);
 *                     workspace: sb_sumsq_workspace_size bytes, zeroed once by the caller
 *   sb_sgd_clip_step  c = min(1, max_norm/(sqrt(sumsq)+1e-6)); [m = momentum*m + c*g]; p -= lr*(m|c*g)
 *                     the clip coefficient is read from device memory (no host sync);
 *                     params_bf16 (may be NULL): bf16 copy of the updated parameters, the
 *                     tensor-core operands of the next step (no per-step cast kernels)
 * ------------------------------------------------------------------------------------- */
int sb_sumsq_workspace_size(size_t* bytes);
int sb_sumsq(const float* g, long long n, float* out, void* workspace, void* stream);
int sb_sgd_clip_step(float* params, const float* grads, float* momentum_buf, void* params_bf16,
                     long long n, const float* sumsq, float lr, float momentum, float max_norm,
                     void* stream);

/* ---------------------------------------------------------------------------------------
 * Attention decoder step of the sequence-to-sequence model (csrc/s2s.cu), fp32.
 * Replaces: the per-token chain nn.Embedding + nn.GRUCell + NNAttention (Conv1d, broadcast add,
 *           ReLU, Linear, softmax, weighted sum) + LinearND of Seq2Seq.decode / decode_step
 *           (speech/models/seq2seq.py:78-137, 344-360) and the host loops of infer (:145-178) and
 *           beam_search (:180-227).
 *   sb_s2s_cell_fwd   ix = emb[tok[b*tok_stride]] + sx_prev (NULL at the first step);
 *                     hx = GRUCell(ix, hx_prev); optionally saves ix and the gates (r, z, n, hn)
 *   sb_s2s_attn_fwd   attention of every row over eh: row b attends over utterance b / eh_group
 *                     (1: its own; the beam search passes K, its rows per utterance), sx (B,H) /
 *                     ax (B,T); with fc_w: logits = fc(hx + sx) written
 *                     at logits[b*logit_stride + c], optional log-softmax, arg-max, greedy history
 *                     and end-token count; `done` (device int, may be NULL): != 0 -> no-op.
 *                     Without fc_w: the attention alone (NNAttention.forward on the decode path)
 *   sb_s2s_dout       backward of the output projection for all (step, utterance) rows at once:
 *                     d_o = dlogits W_fc, o = hx + sx (operand of the time-batched d W_fc)
 *   sb_s2s_attn_bwd / sb_s2s_cell_bwd   gradients of one step (see csrc/s2s.cu)
 *   sb_s2s_check_done greedy stop rule: every row emitted end_tok in the same step
 *   sb_s2s_beam_*     device-side beam bookkeeping with the reference's stable-sort tie order
 * Layouts that differ from the reference's parameters (transposed once per call by the host
 * mirror): conv_wT (Kc, H) = NNAttention.conv.weight (H, 1, Kc) transposed; w_ihT / w_hhT (H, 3H)
 * = GRUCell weights transposed (backward only).  g_conv_wT is (B, ceil(T/24), Kc, H): one slot
 * per CTA, accumulated over the steps, to be summed over its two leading dims by the caller.
 * workspace: >= sb_s2s_workspace_size(B, T, H) bytes, its first 4*B bytes ZERO before the first
 * call (ticket counters; the kernels leave them zero); one workspace serves all steps.
 * Constraints: H % 4 == 0 (attention backward: H <= 1664, its shared-memory tile is 33 H floats),
 * conv kernel width odd and <= 15, T <= 6144, beam <= 32, beam batch B <= 65535.
 * Exact lengths: `lens` (B) int32 on the device gives the frames row b attends over (clamped to
 * [1, T]; NULL = all T).  Frames t >= lens[b] are left out of the softmax, so a_t = 0 exactly
 * there, and out of the location conv's input; log_t scales by log(lens[b]); d eh stays untouched
 * (zero) there.  CTAs whose frame tile lies wholly past lens[b] exit at once.
 * ------------------------------------------------------------------------------------- */
int sb_s2s_workspace_size(int B, int T, int H, size_t* bytes);
int sb_s2s_cell_fwd(const float* emb, const int* tok, int tok_stride, const float* sx_prev,
                    const float* hx_prev, const float* w_ih, const float* w_hh, const float* b_ih,
                    const float* b_hh, float* hx, float* ix_save, float* gates_save,
                    const int* done, int B, int H, void* stream);
int sb_s2s_attn_fwd(const float* eh, int eh_group, const float* hx, const float* ax_prev,
                    const float* conv_wT, const float* conv_b, const float* lin_w, float lin_b,
                    int log_t, int B, int T, int H, int Kc, float* sx, float* ax,
                    const float* fc_w, const float* fc_b, int C, float* logits,
                    long long logit_stride, float* logp, int* argmax, int* history,
                    int hist_stride, int hist_col, int* end_count, int end_tok, const int* done,
                    const int* lens, void* workspace, size_t workspace_bytes, void* stream);
int sb_s2s_dout(const float* dlogits, const float* fc_w, const float* hx, const float* sx,
                float* d_o, float* o_all, long long rows, int C, int H, void* stream);
int sb_s2s_attn_bwd(const float* eh, const float* hx, const float* hx_prev, const float* ax_prev,
                    const float* ax, const float* conv_wT, const float* conv_b,
                    const float* lin_w, const float* d_o, const float* d_ix_next,
                    const float* d_ax_next, const float* d_hx_next, const float* gates,
                    float* d_eh, float* d_ax_prev, float* d_gi, float* d_gh, float* d_hx_direct,
                    float* g_conv_wT, float* g_conv_b, float* g_lin_w, float* g_lin_b, int log_t,
                    int B, int T, int H, int Kc, const int* lens, void* workspace,
                    size_t workspace_bytes, void* stream);
int sb_s2s_cell_bwd(const float* d_gi, const float* d_gh, const float* d_hx_direct,
                    const float* w_ihT, const float* w_hhT, float* d_ix, float* d_hx_prev, int B,
                    int H, void* stream);
int sb_s2s_check_done(const int* end_count, int B, int* done, int* nsteps, int step1, void* stream);
/* Attention rescoring (csrc/s2s_rescore.cu), the second pass of two-pass decoding: R rows, each a
 * hypothesis forced through the step kernels above (row r attends over utterance r / K with
 * eh_group = K).  Row r of tokens (R, ld) int32 is START, y_1 .. y_L with L = lens[r] <= ld - 1
 * (lens (R) int32; L = -1 marks a row that scores nothing, an empty beam slot).
 *   sb_s2s_score_tokens  after step u's log-softmax logp (R, C) float32: acc[r] += (double)
 *       logp[r, y_{u+1}] where u < L, acc[r] += (double) logp[r, end_tok] where u == L, nothing
 *       where u > L.  Called for u = 0, 1, .. in order, acc (R) float64 ends as
 *       a = sum_{u=0..L} (double) l_u, summed in u order, l_u the float32 log-probability of the
 *       u-th forced token; an empty hypothesis (L = 0) scores l(END | START).
 *       Every token read must lie in [0, C) (the caller builds the matrix from
 *       sb_ctc_stream_nbest's labels); the host sees only what it can check.
 * SB_ERR_INVALID for a null pointer, R, C or ld <= 0, u < 0 or end_tok outside [0, C);
 * SB_ERR_UNSUPPORTED for R past 2^31 - 1 blocks of rows.  Both before any CUDA call. */
int sb_s2s_score_tokens(const float* logp, long long R, int C, const int* tokens, int ld,
                        const int* lens, int u, int end_tok, double* acc, void* stream);
/* The beam state is opaque but for the fields the host reads in place: `done` (int32) at byte 0
 * (0 while the search runs, then the number of steps it ran; for one utterance it doubles as the
 * `done` flag of the step kernels), the length of the final hypothesis in out_tokens (int32) at byte 4, and its
 * float64 score in the last 8 bytes of the state.
 * Batched forms (*_batch): B utterances searched at once, each exactly as it would be alone.
 * States [B], nodes [B][node_cap][2], c_scores [B][c_cap], out_tokens [B][max_len + 2] sit back
 * to back; logp, parent_row and tok_next have B*K rows, utterance b's are b*K .. b*K+K-1, and
 * parent_row holds rows within the utterance.  `stop` (device int32[2], zeroed by the init):
 * stop[0] counts the utterances that have stopped, stop[1] becomes 1 when the last one does - the
 * `done` flag of the batch's step kernels.  Rows of stopped utterances are still computed by the
 * step kernels until then; the select and gather of a stopped utterance do nothing.  The
 * single-utterance entry points are the batched ones at B = 1 without `stop`. */
int sb_s2s_beam_state_size(size_t* bytes);
int sb_s2s_beam_init(void* state, int* nodes, int* tok_next, int start_tok, void* stream);
int sb_s2s_beam_select(const float* logp, void* state, double* c_scores, int* nodes,
                       int* parent_row, int* tok_next, int* out_tokens, int K, int C, int end_tok,
                       int step, int max_len, int node_cap, int c_cap, void* stream);
int sb_s2s_beam_gather(const float* hx_in, const float* sx_in, const float* ax_in, float* hx_out,
                       float* sx_out, float* ax_out, const int* parent_row, const void* state,
                       int K, int H, int T, void* stream);
int sb_s2s_beam_init_batch(void* state, int* nodes, int node_cap, int* tok_next, int K,
                           int start_tok, int* stop, int B, void* stream);
int sb_s2s_beam_select_batch(const float* logp, void* state, double* c_scores, int* nodes,
                             int* parent_row, int* tok_next, int* out_tokens, int K, int C,
                             int end_tok, int step, int max_len, int node_cap, int c_cap,
                             int* stop, int B, void* stream);
int sb_s2s_beam_gather_batch(const float* hx_in, const float* sx_in, const float* ax_in,
                             float* hx_out, float* sx_out, float* ax_out, const int* parent_row,
                             const void* state, int K, int H, int T, int B, void* stream);

/* Large vocabularies (csrc/s2s_vocab.cu, csrc/s2s.cu).  sb_s2s_attn_fwd runs the output projection
 * in the utterance's last CTA, which holds every logit in shared memory: it takes fc_w only where
 * sb_s2s_fc_fused(H, C) is 1 (C <= 7 H; pure host arithmetic).  Other shapes run the attention
 * without fc_w, then:
 *   sb_s2s_fc_rows    logits of R rows over many CTAs: o = hx + sx (sx may be NULL), row r written
 *                     at logits + (r % row_group) * ld0 + (r / row_group) * ld1 (logits may be
 *                     NULL); each logit is summed in an order that depends on H only, so a row
 *                     projects to the same bits alone or among any number of rows.  The same launch
 *                     reduces every row (deterministic, in-kernel tickets): optional arg-max (first
 *                     maximum), greedy history[r * hist_stride + hist_col], end_count += 1 where
 *                     the arg-max is end_tok, and the row's log-sum-exp, kept in the workspace
 *   sb_s2s_fc_logp    logp (R, C) = logits - log-sum-exp of the last sb_s2s_fc_rows on the same
 *                     workspace and shape (logp may alias a dense logits buffer)
 *   workspace: >= sb_s2s_fc_workspace_size(R, C) bytes, ZERO before the first call; one workspace
 *   serves every call with the same (R, C) on one stream.  H % 4 == 0, H <= 3200.
 * The single-CTA sb_s2s_beam_select holds all K*C float64 candidates in shared memory:
 * sb_s2s_beam_select_fits(K, C) is 1 where it runs (K <= 32, K*C*8 <= 200 KB).  Otherwise
 *   sb_s2s_beam_select_split  the same selection and bookkeeping (same state, outputs and tie
 *                     order) in two stages: per-tile top 2K candidates over many CTAs, then one
 *                     CTA merges the tiles' lists; workspace >= sb_s2s_beam_split_workspace_size
 *                     (batched: sb_s2s_beam_split_workspace_size_batch, B times as many bytes).
 * Backward of the projection where sb_s2s_dout does not run (C > 8192): d_o = dlogits W_fc as a
 * 3-pass split-bf16 sb_gemm_bf16_tn with SB_GEMM_B_MN (the host mirror, functions/s2s.py). */
int sb_s2s_fc_fused(int H, int C);
int sb_s2s_fc_workspace_size(long long R, int C, size_t* bytes);
int sb_s2s_fc_rows(const float* hx, const float* sx, const float* fc_w, const float* fc_b,
                   long long R, int H, int C, float* logits, int row_group, long long ld0,
                   long long ld1, int* argmax, int* history, int hist_stride, int hist_col,
                   int* end_count, int end_tok, const int* done, void* workspace,
                   size_t workspace_bytes, void* stream);
int sb_s2s_fc_logp(const float* logits, int row_group, long long ld0, long long ld1, float* logp,
                   long long R, int C, const int* done, const void* workspace,
                   size_t workspace_bytes, void* stream);
int sb_s2s_beam_select_fits(int K, int C);
int sb_s2s_beam_split_workspace_size(int K, int C, size_t* bytes);
int sb_s2s_beam_select_split(const float* logp, void* state, double* c_scores, int* nodes,
                             int* parent_row, int* tok_next, int* out_tokens, int K, int C,
                             int end_tok, int step, int max_len, int node_cap, int c_cap,
                             void* workspace, size_t workspace_bytes, void* stream);
int sb_s2s_beam_split_workspace_size_batch(int K, int C, int B, size_t* bytes);
int sb_s2s_beam_select_split_batch(const float* logp, void* state, double* c_scores, int* nodes,
                                   int* parent_row, int* tok_next, int* out_tokens, int K, int C,
                                   int end_tok, int step, int max_len, int node_cap, int c_cap,
                                   int* stop, int B, void* workspace, size_t workspace_bytes,
                                   void* stream);

/* Attention beam search with shallow fusion of the n-gram LM (SbNgramLm above).
 *   sb_s2s_beam_select_lm_batch        sb_s2s_beam_select_batch with the LM and its weights
 *   sb_s2s_beam_select_split_lm_batch  sb_s2s_beam_select_split_batch with the LM and its weights
 * Candidate (r, c), live row r extended by class c, has the float64 value
 *   score_r + ((double)logp[r][c] + (lm_weight * lm(c | h_r) + beta_c)),
 * evaluated in that order, with beta_c = insertion_bonus for c != end_tok and 0 for end_tok.  h_r
 * is row r's last order-1 tokens; its root (the start token) reads as <s>, before which there is
 * nothing.  The fused values are the hypothesis scores throughout: selection, completion, the stop
 * rule and the final score.  With lm_weight = insertion_bonus = 0 the results equal the LM-less
 * entry points' bit for bit.  The LM's classes are the model's vocabulary: lm->tok[end_tok] must
 * be the token of </s> (the ABI cannot check this; speech_b200.lm.NGramLM with `end` builds such
 * tables), and lm->blank is the start token, which must not be a class the search scores.
 * SB_ERR_INVALID for a null LM or table pointer, lm_weight < 0, a non-finite weight or bound,
 * lm->num_classes < C, 0 <= lm->blank < C, or a cap that is not a power of two;
 * SB_ERR_UNSUPPORTED for order > SB_LM_MAX_ORDER; otherwise as the LM-less entry points. */
int sb_s2s_beam_select_lm_batch(const float* logp, void* state, double* c_scores, int* nodes,
                                int* parent_row, int* tok_next, int* out_tokens, int K, int C,
                                int end_tok, int step, int max_len, int node_cap, int c_cap,
                                int* stop, int B, const SbNgramLm* lm, double lm_weight,
                                double insertion_bonus, void* stream);
int sb_s2s_beam_select_split_lm_batch(const float* logp, void* state, double* c_scores,
                                      int* nodes, int* parent_row, int* tok_next, int* out_tokens,
                                      int K, int C, int end_tok, int step, int max_len,
                                      int node_cap, int c_cap, int* stop, int B, void* workspace,
                                      size_t workspace_bytes, const SbNgramLm* lm,
                                      double lm_weight, double insertion_bonus, void* stream);

/* Attention beam search with a word n-gram LM (SbWordLm below): the CTC word-LM contract moved onto
 * the attention search's candidates.
 *   sb_s2s_beam_select_wordlm_batch        sb_s2s_beam_select_batch with the LM, its three weights
 *                                          and word_nodes
 *   sb_s2s_beam_select_split_wordlm_batch  sb_s2s_beam_select_split_batch with the same
 *   sb_s2s_ctc_candidates_wordlm           sb_s2s_ctc_candidates with the same (joint search)
 * Candidate (r, c), live row r extended by class c, with p = (double)logp[r][c] and score_r the
 * row's float64 score, is valued (float64, in this order):
 *   c the delimiter, n_r = 0:      score_r + p (leading and repeated delimiters are free);
 *   c the delimiter, n_r != 0:     score_r + (p + d_r), d_r = (lm_weight * lm(w | hist_r) +
 *       insertion_bonus) + g_r exactly as in the CTC search: w the word at n_r, or <unk>; g_r =
 *       oov_penalty where n_r >= 1 is not a word, else 0;
 *   c = end_tok:                   score_r + (p + t_r), t_r = e_r + lm_weight * lm(</s> | hist'_r),
 *       e_r = d_r, or 0.0 for an empty partial word, hist'_r the history with the trailing word
 *       (the CTC search's end-of-utterance term);
 *   any other c, n_r >= 0 with no lexicon child c:  score_r + (p + oov_penalty), the new row's node
 *       -1;
 *   any other c otherwise:         score_r + p.
 * n_r is row r's lexicon node (0 the empty partial word; -1 the partial word has left the lexicon,
 * its OOV penalty already charged); hist_r its last order-1 completed words, <s> before the first;
 * the start token begins the history and spells nothing.  The fused value is the hypothesis score
 * everywhere after: selection, the "first K may complete" rule, the stop rule, the chosen
 * hypothesis and the returned score, which for a completed hypothesis is acoustic + lm_weight *
 * (word LM with </s>) + insertion_bonus * words + oov_penalty * OOV words; a hypothesis returned
 * live at max_len has no end term.  With lm_weight = insertion_bonus = oov_penalty = 0 the results
 * equal the LM-less entry points' bit for bit.  Candidates valued -inf (oov_penalty = -inf) are
 * ordinary values under the usual tie order.  In the joint search the LM part of P(r, c) is the
 * term above (d_r, t_r, oov_penalty or 0) in place of lm_weight * lm(c | h_r) + beta_c.
 * The LM's classes are the model's: lm->blank is the start token, no class the search scores, and
 * end_tok is the LM's end class (speech_b200.lm.WordLM with `end` builds such tables).
 * word_nodes: device int32 [B][node_cap][3], parallel to nodes, no initial contents needed: each
 * step writes the word state of every live row's node (lexicon node, last completed word token or
 * -1, a node holding the words before it), computed from its parent's with at most one lexicon
 * probe, and reads the history up those links; a row's cost is O(order) probes, independent of the
 * length of its words.  The same buffer must serve every step of a search.
 * SB_ERR_INVALID for a null table or word_nodes, lm_weight < 0 or not finite, insertion_bonus not
 * finite, oov_penalty > 0 or NaN, oov_penalty != -inf without <unk>, lm->num_classes < C, lm->blank
 * in [0, C), a delimiter outside [0, C) or equal to end_tok, a cap that is not a power of two, or
 * order < 1; SB_ERR_UNSUPPORTED for order > SB_LM_MAX_ORDER or K > 32; otherwise as the LM-less
 * entry points.  All before any CUDA call. */
int sb_s2s_beam_select_wordlm_batch(const float* logp, void* state, double* c_scores, int* nodes,
                                    int* parent_row, int* tok_next, int* out_tokens, int K, int C,
                                    int end_tok, int step, int max_len, int node_cap, int c_cap,
                                    int* stop, int B, const SbWordLm* lm, double lm_weight,
                                    double insertion_bonus, double oov_penalty, int* word_nodes,
                                    void* stream);
int sb_s2s_beam_select_split_wordlm_batch(const float* logp, void* state, double* c_scores,
                                          int* nodes, int* parent_row, int* tok_next,
                                          int* out_tokens, int K, int C, int end_tok, int step,
                                          int max_len, int node_cap, int c_cap, int* stop, int B,
                                          void* workspace, size_t workspace_bytes,
                                          const SbWordLm* lm, double lm_weight,
                                          double insertion_bonus, double oov_penalty,
                                          int* word_nodes, void* stream);

/* Joint CTC/attention decoding of the attention model (Watanabe et al. 2017, Algorithm 2;
 * csrc/s2s_ctc.cu): the batched beam search above with the CTC prefix scores of a CTC head.
 * y (B, T, C) float32: the head's log-probabilities, C = the decoder's classes, blank C - 1, which
 * is also end_tok; start_tok = C.  lambda = ctc_weight in (0, 1); M in [1, min(C, 128)] candidates
 * per live row; lens (B) frames of each utterance (clamped to [1, T]) or null (all T).
 * Per live row r the search keeps A_r (attention + LM part), psi_r = psi(h_r) and the CTC forward
 * variables gn_t(h_r), gb_t(h_r), t < T_b; its score is S_r = A_r + lambda psi_r, used for
 * selection, completion, the stop rule and the result.  The root has A = psi = 0, gn = -inf,
 * gb_t = sum_{tau <= t} y_tau(blank).
 *   P(r, c) = (1 - lambda) (double)logp[r][c] (+ (lm_weight lm(c | h_r) + beta_c) with an LM, as
 *   in the LM entry points); row r's candidates are its M classes with the largest P (ties to the
 *   lower class), in class order; value = (A_r + P) + lambda psi(h_r + c), in float64.
 *   psi(h + END) = log(exp gn_{T_b-1}(h) + exp gb_{T_b-1}(h)); for a label c: gn_0(h + c) = y_0(c)
 *   at the root, else -inf; gb_0 = -inf; psi = gn_0; for t = 1..T_b-1, Phi = gb_{t-1}(h) when c
 *   is h's last label, else lse(gb_{t-1}(h), gn_{t-1}(h)); gn_t = lse(gn_{t-1}, Phi) + y_t(c);
 *   gb_t = lse(gb_{t-1}, gn_{t-1}) + y_t(blank); psi = lse(psi, Phi + y_t(c)); lse(a, b) =
 *   max + log1p(exp(min - max)), -inf when both are.
 * Selection: the first min(2K, nl M) candidates by (value desc, (r, c) asc), and the bookkeeping
 * of sb_s2s_beam_select_batch; a new live row gets A' = A_r + P and psi' = psi(h_r + c).
 *   sb_s2s_ctc_state_size    bytes of the CTC buffer, R = B*K rows, carved in this order:
 *                            A [R] double; the vectors [2][R][2][T] double (gn then gb of each
 *                            row, buffer (step & 1) holding the rows entering step `step`); the
 *                            rows' candidate lists [R][M] double values, [R][M] double A_r + P,
 *                            [R][M] double psi(h_r + c), [R][M] int classes (ascending)
 *   sb_s2s_ctc_init          after sb_s2s_beam_init_batch: every utterance's root
 *   sb_s2s_ctc_candidates    per step after the attention step's logp: the rows' candidate lists;
 *                            lm optional (null: lm_weight = insertion_bonus = 0), checked as in
 *                            the LM entry points; a no-op once stop[1] is set
 *   sb_s2s_ctc_select_batch  per step: selection, bookkeeping, the new rows' A (one CTA per
 *                            utterance), then their vectors (one thread per new row); then
 *                            sb_s2s_beam_gather_batch as usual
 * SB_ERR_INVALID for a null pointer, K, T, B < 1, C < 2, M outside [1, C], lambda outside (0, 1),
 * end_tok != C - 1 or start_tok != C; SB_ERR_UNSUPPORTED for K > 32, M > 128, B > 65535, or
 * (candidates) C > 20480; SB_ERR_WORKSPACE for a CTC buffer below sb_s2s_ctc_state_size. */
int sb_s2s_ctc_state_size(int K, int M, int T, int B, size_t* bytes);
int sb_s2s_ctc_init(const float* ctc_logp, const int* lens, void* ctc_state,
                    size_t ctc_state_bytes, int K, int C, int M, int T, int start_tok, int end_tok,
                    double ctc_weight, int B, void* stream);
int sb_s2s_ctc_candidates(const float* logp, const float* ctc_logp, const int* lens,
                          const void* state, const int* nodes, int node_cap, void* ctc_state,
                          size_t ctc_state_bytes, int K, int C, int M, int T, int start_tok,
                          int end_tok, double ctc_weight, int step, const int* stop, int B,
                          const SbNgramLm* lm, double lm_weight, double insertion_bonus,
                          void* stream);
int sb_s2s_ctc_candidates_wordlm(const float* logp, const float* ctc_logp, const int* lens,
                                 const void* state, const int* nodes, int node_cap,
                                 void* ctc_state, size_t ctc_state_bytes, int K, int C, int M,
                                 int T, int start_tok, int end_tok, double ctc_weight, int step,
                                 const int* stop, int B, const SbWordLm* lm, double lm_weight,
                                 double insertion_bonus, double oov_penalty, int* word_nodes,
                                 void* stream);
int sb_s2s_ctc_select_batch(const float* ctc_logp, const int* lens, void* ctc_state,
                            size_t ctc_state_bytes, void* state, double* c_scores, int* nodes,
                            int* parent_row, int* tok_next, int* out_tokens, int K, int C, int M,
                            int T, int start_tok, int end_tok, double ctc_weight, int step,
                            int max_len, int node_cap, int c_cap, int* stop, int B, void* stream);

/* ---------------------------------------------------------------------------------------
 * RNN-Transducer loss + gradient w.r.t. the log-probabilities.
 * Replaces: transducer.functions.transducer.TransducerLoss()(log_probs, labels, x_lens, y_lens)
 *           (libs/transducer, un-vendored, Makefile:10-12; call site
 *            speech/models/transducer_model.py:46-52).
 *   log_probs (B, T, U1, V) float32 log-softmax over V (U1 = max label length + 1)
 *   grads     same shape, out (zero-filled here, then the 2 non-zero entries per cell); may be NULL
 *   labels    flat int32; label_offsets exclusive prefix sum; label_lens (B); act_lens (B)
 *   blank     blank class index (reference: V-1, transducer_model.py:28)
 *   costs     (B) float32 out
 * ------------------------------------------------------------------------------------- */
int sb_rnnt_workspace_size(int B, int T, int U1, size_t* bytes);
int sb_rnnt_fwd_bwd(const float* log_probs, float* grads, const int* labels,
                    const int* label_offsets, const int* label_lens, const int* act_lens, int B,
                    int T, int U1, int V, int blank, float* costs, void* workspace,
                    size_t workspace_bytes, void* stream);

/* Compact-lattice form of the same loss: `lat` / `garc` are (T, B, U1, 2), TIME-major nodes
 * n = (t*B + b)*U1 + u, = {log p(blank), log p(label of arc u -> u+1)} per node (what
 * sb_rnnt_joint_fwd writes) and the gradients w.r.t. them. */
int sb_rnnt_fwd_bwd_compact(const float* lat, float* garc, const int* labels,
                            const int* label_offsets, const int* label_lens, const int* act_lens,
                            int B, int T, int U1, int blank, float* costs, void* workspace,
                            size_t workspace_bytes, void* stream);

/* Transducer Viterbi (forced) alignment over the same compact lattice (csrc/rnnt.cu): the single
 * best path, in float64,
 *   a[0][0] = 0,  a[t][u] = max(a[t-1][u] + blank(t-1, u), a[t][u-1] + label(t, u-1)),
 *   score = a[T_b-1][U_b] + blank(T_b-1, U_b).
 * Tie rule: where the two arcs into (t, u) score equal, the max takes the blank arc from (t-1, u),
 * i.e. the path on which label u-1 was emitted at an earlier frame; read back from (T_b-1, U_b),
 * each label is thus emitted at the earliest frame among equal paths, the last label first (on a
 * lattice of equal values every label is emitted at frame 0).  Shapes as sb_rnnt_fwd_bwd_compact
 * (U1 <= 1024); the labels are not read.
 *   frames   (B, U1-1) int32 out: the frame at which label u is emitted; -1 past U_b, and
 *            everywhere when the score is -inf
 *   scores   (B) float64 out: the path's log-probability; -inf where act_lens[b] = 0
 *   workspace >= sb_rnnt_viterbi_workspace_size(...) bytes: 1-bit backpointers by anti-diagonal,
 *            B * (T + U1) * ceil(U1 / 256) * 32 bytes (the count rounded up to 1, 2 or 4), + 256.
 * SB_ERR_INVALID for a NULL pointer or B, T, U1 <= 0; SB_ERR_UNSUPPORTED for U1 > 1024; both
 * before any launch. */
int sb_rnnt_viterbi_workspace_size(int B, int T, int U1, size_t* bytes);
int sb_rnnt_viterbi(const float* lat, const int* labels, const int* label_offsets,
                    const int* label_lens, const int* act_lens, int B, int T, int U1, int* frames,
                    double* scores, void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------
 * Fused RNN-T joint network: relu(fx[b,t,:] + fy[b,u,:]) -> fc2 -> log-softmax per lattice node,
 * the (B, T', U+1, H) intermediate never exists (it lives as 16 KB operand tiles in shared memory).
 * Replaces: the broadcast add + ReLU + LinearND + log_softmax of Transducer.decode,
 *           speech/models/transducer_model.py:71-76 (fc1 shared by both streams, :73).
 *   fx [B*T][H] f32 = fc1(encoder states), fy [B*U1][H] f32 = fc1(prediction network) (biases in)
 *   w2 [V1][H] bf16, b2 [V1] f32: fc2;  ymat [B][U1-1] int32 end-padded labels
 *   node order of lat / garc / dlogits: TIME-major, n = (t*B + b)*U1 + u (frames t0..t0+Tc-1
 *   are one contiguous slab of rows)
 *   sb_rnnt_joint_fwd:      lat [nodes][2] (out), lp_full (B, T, U1, V1) batch-first (out, may be
 *                           NULL: only `infer` needs every class)
 *   sb_rnnt_joint_dlogits:  backward recompute pass: garc [nodes][2] (gradient w.r.t. lat) ->
 *                           dlogits [nodes][NV] bf16 (NV = 32 if V1 <= 32 else 64), db2 [V1] +=
 *   sb_rnnt_joint_build_slab / _reduce_slab: the hidden activations of Tc <= 8 frames
 *                           (z [B*Tc*U1][H] bf16) for the weight-gradient GEMMs, and the masked
 *                           reduction of dz [B*Tc*U1][H] f32 into dfx (=) and dfy (+=)
 * Constraints: H % 8 == 0, V1 <= 64, and fc2's weight must fit in shared memory next to the
 * operand ring (H <= 1792 for V1 <= 32, H <= 1024 for V1 <= 64): sb_rnnt_joint_resident(H, V1)
 * answers 1 exactly for the shapes sb_rnnt_joint_fwd / _dlogits run (pure host arithmetic).  Every
 * other shape goes through the slab path below: build_slab, sb_gemm_bf16_tn for the logits, and
 * sb_rnnt_joint_vocab_fwd_rows / _bwd_rows.
 * ------------------------------------------------------------------------------------- */
int sb_rnnt_joint_resident(int H, int V1);
int sb_rnnt_joint_fwd(const float* fx, const float* fy, const void* w2_bf16, const float* b2,
                      const int* ymat, float* lat, float* lp_full, int B, int T, int U1, int H,
                      int V1, int blank, void* stream);
int sb_rnnt_joint_dlogits(const float* fx, const float* fy, const void* w2_bf16, const float* b2,
                          const int* ymat, const float* garc, void* dlogits_bf16, float* db2, int B,
                          int T, int U1, int H, int V1, int blank, void* stream);
int sb_rnnt_joint_build_slab(const float* fx, const float* fy, void* z_bf16, int B, int T, int U1,
                             int H, int t0, int Tc, void* stream);
int sb_rnnt_joint_reduce_slab(const float* dz, const void* z_bf16, float* dfx, float* dfy, int B,
                              int T, int U1, int H, int t0, int Tc, void* stream);

/* ---------------------------------------------------------------------------------------
 * Row kernels of the large-vocabulary joint (any V1; the models use them for V1 > 64, where fc2's
 * weight does not fit the shared memory of the fused kernel).  The caller walks the lattice a slab
 * of Tc frames at a time: z = sb_rnnt_joint_build_slab, logits = z W2^T + b2 with sb_gemm_bf16_tn
 * into f32 rows [Tc*B*U1][ld]; row r of the slab is node n = t0*B*U1 + r.
 *   sb_rnnt_joint_vocab_fwd_rows: per row, max and log-sum-exp over the first V1 columns ->
 *       lat [nodes][2] = {v_blank - lse, v_label - lse} (label -inf at u = U1-1, as
 *       sb_rnnt_joint_fwd), lse [nodes] (kept for the backward pass), and, if lp_full is not NULL,
 *       the slab's rows of the batch-first (B, T, U1, V1) log-probabilities.
 *   sb_rnnt_joint_vocab_bwd_rows: from the recomputed logits, lse and garc [nodes][2] ->
 *       dlogits [Tc*B*U1][ldd] bf16, dlogit_k = g_b [k = blank] + g_l [k = label]
 *       - (g_b + g_l) exp(v_k - lse), zero in columns V1 .. ldd-1;  db2 [V1] += its column sums.
 * lat, lse and garc are the whole-lattice arrays (indexed by n), logits / dlogits the slab's rows.
 * Constraints: 0 <= blank < V1, 0 <= t0, t0 + Tc <= T, ld and ldd >= V1 and multiples of 8,
 * logits and dlogits 16-byte aligned.
 * ------------------------------------------------------------------------------------- */
int sb_rnnt_joint_vocab_fwd_rows(const float* logits, long long ld, const int* ymat, float* lat,
                                 float* lse, float* lp_full, int B, int T, int U1, int V1, int blank,
                                 int t0, int Tc, void* stream);
int sb_rnnt_joint_vocab_bwd_rows(const float* logits, long long ld, const float* lse,
                                 const float* garc, const int* ymat, void* dlogits_bf16,
                                 long long ldd, float* db2, int B, int T, int U1, int V1, int blank,
                                 int t0, int Tc, void* stream);
/* Shortlists of the lattice for sb_rnnt_decode_static_shortlist, one per node, batch-first:
 *   sl_val  (B, T, U1, kp) f32  the kp best non-blank lp by (lp desc, class asc), -inf padded
 *   sl_idx  (B, T, U1, kp) i32  their classes, -1 past the V1 - 1 non-blank classes
 *   sl_meta (B, T, U1, 2)  f32  {lp of the blank, lp of the (kp+1)-th non-blank class or -inf}
 * lp_k = v_k - lse[n] in the fp32 arithmetic of sb_rnnt_joint_vocab_fwd_rows' lp_full (bit-
 * identical values), or v_k itself when lse is NULL.  Rows of v (leading dimension ld >= V1, any
 * alignment) are either
 *   time_major = 1: a slab of the joint, as sb_rnnt_joint_vocab_fwd_rows reads it (row r is node
 *                   n = t0*B*U1 + r; lse indexed by n), or
 *   time_major = 0: the whole batch-first (B, T, U1) lattice (t0 = 0, Tc = T).
 * 1 <= kp <= 64 (SB_ERR_UNSUPPORTED above). */
int sb_rnnt_shortlist_rows(const float* v, long long ld, const float* lse, int B, int T, int U1,
                           int V1, int blank, int kp, int t0, int Tc, int time_major,
                           float* sl_val, int* sl_idx, float* sl_meta, void* stream);

/* ---------------------------------------------------------------------------------------
 * Transducer beam search over a precomputed (teacher-forced) lattice, one CTA per utterance.
 * Replaces: transducer.decoders.decode_static(lp, beam_size, blank) of the un-vendored
 *           awni/transducer, called per utterance on a host array at
 *           speech/models/transducer_model.py:92-101.
 *   lp       (B, T, U1, V) f32 log-probabilities (device)
 *   tlens    (B) frames searched per utterance, ulens (B) lattice rows (labels + 1)
 *   out_labels (B, U1) int32, out_lens (B), out_scores (B) f64 log-probability of the best
 *   workspace >= sb_rnnt_decode_static_workspace_size bytes;  beam_size <= 32
 * sb_rnnt_decode_static keeps every candidate in shared memory: it runs where
 * beam_size * V * 8 + 16 <= 200 KB, which sb_rnnt_decode_static_fits(beam_size, V) answers (1 / 0,
 * host arithmetic); SB_ERR_UNSUPPORTED elsewhere.
 * sb_rnnt_decode_static_shortlist runs the same search, at any V, from the shortlists of
 * sb_rnnt_shortlist_rows (kp per node, beam_size <= kp <= 64): a K-way merge of the frontier's
 * lists replaces the scan of beam_size * V candidates.  Labels, lengths and scores are bit-
 * identical to sb_rnnt_decode_static unless out_flags (B, int32) counts, for an utterance, a
 * selection the lists cannot prove (two distinct float32 lp rounding to one float64 score at the
 * end of a list, csrc/tdecode.cu); rerun such utterances with longer lists.
 * ------------------------------------------------------------------------------------- */
int sb_rnnt_decode_static_workspace_size(int B, int T, int U1, int beam_size, size_t* bytes);
int sb_rnnt_decode_static_fits(int beam_size, int V);
int sb_rnnt_decode_static(const float* lp, const int* tlens, const int* ulens, int B, int T, int U1,
                          int V, int beam_size, int blank, int* out_labels, int* out_lens,
                          double* out_scores, void* workspace, size_t workspace_bytes,
                          void* stream);
int sb_rnnt_decode_static_shortlist(const float* sl_val, const int* sl_idx, const float* sl_meta,
                                    int kp, const int* tlens, const int* ulens, int B, int T,
                                    int U1, int V, int beam_size, int blank, int* out_labels,
                                    int* out_lens, double* out_scores, int* out_flags,
                                    void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------
 * Label-free transducer beam search (csrc/rnnt_search.cu): the search above with the row of
 * hypothesis h at frame t computed from h itself (prediction network run on h's labels) instead of
 * read at lat[t, len(h)].  The caller's loop, per frame t and level l = 0 .. S
 * (S = max_symbols_per_frame): rows of the level-l frontier, sb_rnnt_search_round, and for l < S
 * the prediction states of the new frontier; then sb_rnnt_search_frame_end.  Once before:
 * sb_rnnt_search_init; once after: sb_rnnt_search_final.  Each call is one launch, one CTA per
 * utterance; utterances with t >= tlens[b] (or no live frontier) return at once.
 *   workspace  >= sb_rnnt_search_workspace_size(B, T, S, beam_size) bytes =
 *              1024 + 4096 + B * (1184 + 8 n + 12 c + 20 d) with n = T*S*K + 2 trie nodes,
 *              c = the least power of two >= max(64, 2 n) map slots, d = K*(S+1) + 1 `done` entries
 *   slot_lens  (B, K) int32: labels of the hypothesis in each slot of the frontier whose rows are
 *              asked for next (what a static lattice needs to supply rows)
 *   sb_rnnt_search_round: rows of the level's K frontier slots, either lp (B, K, V) f32 (needs
 *              beam_size * V * 8 + 16 <= 200 KB, sb_rnnt_decode_static_fits) or, with lp NULL, the
 *              shortlists (B, K, kp) / (B, K, 2) of sb_rnnt_shortlist_rows; writes par (B, K) the
 *              parent slot of each new frontier slot (-2: none), sym (B, K) its symbol, slot_lens
 *   sb_rnnt_search_frame_end: the K best of `done` become the beam; when hid / fy are not NULL it
 *              gathers their prediction states into block `next` of the arenas hid [S+2][layers]
 *              [B*K][H] and fy [S+2][B*K][Hj] (block l = level l's frontier, blocks cur / next =
 *              0 / S+1 in turn = the beam)
 *   sb_rnnt_search_final: out_labels (B, max_len), out_lens, out_scores (f64), out_flags (may be
 *              NULL; shortlist selections the lists could not prove, as in
 *              sb_rnnt_decode_static_shortlist)
 * sb_rnnt_pred_step: one GRU layer (gates r, z, n; fp32 on CUDA cores) over R = B*K rows: input row
 *   emb[sym[r]] (Kin = embedding width; sym[r] = -1 or sym NULL: zeros) or x[r] (Kin = H), hidden
 *   state h_prev[(r / K) * K + par[r]] (par[r] = -1 or par NULL: zeros; -2: row skipped) -> h[r],
 *   and bf16(h[r]) at y[r * ldy] if y is not NULL.  beam_size <= 32, kp <= 64.
 * Streaming (speech_b200.streaming.TransducerStream): the same entry points resume a search across
 * calls.  The workspace is sized and every call is made with T = max_frames, the most frames a
 * stream is ever searched over (T only sizes the workspace's carve: trie node ids come from each
 * utterance's own count of selection rounds, never from t); each push of n_b new frames runs the
 * loop above for t = 0 .. max_b n_b - 1, local to the push, with tlens = the n_b, so that stream b
 * takes its n_b frames and is left untouched by the others.  sb_rnnt_search_final does not change
 * the state: it may be read after any push.  Default workspace, K = 8, S = 4, max_frames = 3000:
 * 5120 + B * 3,915,748 bytes (about 3.7 MiB per stream).
 * sb_rnnt_search_reset: utterances [first, first + count) back to sb_rnnt_search_init's state
 *   (the empty hypothesis at frame 0: cleared trie, the root as the beam, zero counters and flag,
 *   slot_lens rows zero), others untouched; sb_rnnt_search_init is the reset of [0, B).
 *   SB_ERR_INVALID for a null slot_lens or workspace, bad sizes or a range outside [0, B),
 *   SB_ERR_WORKSPACE for a short workspace, SB_ERR_UNSUPPORTED for beam_size > 32.
 * ------------------------------------------------------------------------------------- */
int sb_rnnt_search_workspace_size(int B, int T, int S, int beam_size, size_t* bytes);
int sb_rnnt_search_init(int* slot_lens, int B, int T, int S, int beam_size, void* workspace,
                        size_t workspace_bytes, void* stream);
int sb_rnnt_search_reset(int* slot_lens, int B, int T, int S, int beam_size, int first, int count,
                         void* workspace, size_t workspace_bytes, void* stream);
int sb_rnnt_search_round(const float* lp, const float* sl_val, const int* sl_idx,
                         const float* sl_meta, int kp, const int* tlens, int t, int level,
                         int max_len, int* par, int* sym, int* slot_lens, int B, int T, int S,
                         int V, int beam_size, int blank, void* workspace, size_t workspace_bytes,
                         void* stream);
int sb_rnnt_search_frame_end(const int* tlens, int t, int* slot_lens, float* hid, int layers,
                             int H, float* fy, int Hj, int cur, int next, int B, int T, int S,
                             int beam_size, void* workspace, size_t workspace_bytes, void* stream);
int sb_rnnt_search_final(int* out_labels, int max_len, int* out_lens, double* out_scores,
                         int* out_flags, int B, int T, int S, int beam_size, void* workspace,
                         size_t workspace_bytes, void* stream);
int sb_rnnt_pred_step(const float* emb, const int* sym, const float* x, const float* h_prev,
                      const int* par, const float* w_ih, const float* w_hh, const float* b_ih,
                      const float* b_hh, float* h, void* y_bf16, int ldy, int R, int K, int Kin,
                      int H, void* stream);

/* Label-free transducer beam search with shallow fusion of the n-gram LM (SbNgramLm above).
 * The LM's classes are the model's: labels and the blank, no end class.  Per level the caller
 * enqueues, after the acoustic rows lp (B, K, V) f32 of the frontier slots:
 *   sb_rnnt_search_lm_rows   per live frontier slot (a workspace of the same search, read for the
 *                            slots' hypotheses) the fused float64 values
 *                              f_k = (double)lp_k + (lm_weight * lm(k | h) + insertion_bonus)
 *                            for every label k, evaluated in that order, and f_blank = (double)
 *                            lp_blank; written either as rows fused (B, K, V) f64 (full route) or,
 *                            with fused NULL, as the kp best by (f desc, k asc): sl_val (B, K, kp)
 *                            f64, sl_idx (B, K, kp) int32 (-inf / -1 padded) and sl_meta (B, K, 2)
 *                            f64 = {f_blank, the (kp+1)-th f or -inf}
 *   sb_rnnt_search_round_lm  sb_rnnt_search_round over those f64 rows or lists (same arguments)
 * h is the hypothesis's last order-1 labels, preceded by <s> where it is shorter (the trie's root
 * reads as <s>); there is no end-of-sentence term.  A blank emission scores score + f_blank; the
 * fused values are the scores throughout: the selections, the merges into `done`, the next beam
 * and out_scores of sb_rnnt_search_final.  With lm_weight = insertion_bonus = 0 the results equal
 * the LM-less search's bit for bit.
 * sb_rnnt_search_lm_rows returns SB_ERR_INVALID for a null LM or table pointer, lm_weight < 0, a
 * non-finite weight or bound, lm->num_classes < V, lm->blank != blank, a cap that is not a power
 * of two, or what sb_rnnt_search_round rejects (kp < beam_size on the shortlist route included);
 * SB_ERR_UNSUPPORTED for order > SB_LM_MAX_ORDER or kp > 64.  sb_rnnt_search_round_lm returns
 * what sb_rnnt_search_round returns. */
int sb_rnnt_search_lm_rows(const float* lp, double* fused, double* sl_val, int* sl_idx,
                           double* sl_meta, int kp, const int* tlens, int t, int level, int B,
                           int T, int S, int V, int beam_size, int blank, const SbNgramLm* lm,
                           double lm_weight, double insertion_bonus, void* workspace,
                           size_t workspace_bytes, void* stream);
int sb_rnnt_search_round_lm(const double* lp, const double* sl_val, const int* sl_idx,
                            const double* sl_meta, int kp, const int* tlens, int t, int level,
                            int max_len, int* par, int* sym, int* slot_lens, int B, int T, int S,
                            int V, int beam_size, int blank, void* workspace,
                            size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Scoring (SURVEY.md section 8f rank 4), HOST function: Levenshtein distance of two int32 token
 * sequences; replaces `editdistance.eval` in speech/utils/score.py:15-16.  Returns -1 on invalid
 * arguments. */
long long sb_edit_distance(const int* a, long long na, const int* b, long long nb);

/* ---------------------------------------------------------------------------------------------
 * Featuriser (SURVEY.md section 8f rank 2).  Replaces speech/loader.py:152-166 `log_specgram`
 * (scipy.signal.spectrogram, periodic Hann window, one-sided density PSD, no detrend / padding,
 * then log(float32(PSD) + eps)) and the normalisation of loader.py:65-67 `(x - mean) / std`.
 *   pcm        int16 samples of all utterances, concatenated (device)
 *   offsets    [B] index of each utterance's first sample in pcm (device, int64)
 *   n_samples  [B] samples per utterance (device, int32)
 *   nperseg    window length in samples (<= 1024), step = nperseg - noverlap
 *   scale      1 / (sample_rate * sum(window^2)), computed by the caller in float64
 *   mean, stdev [nperseg/2+1] per-bin statistics (device, float32) or NULL for the raw log PSD
 *   out        [B][max_frames][nperseg/2+1] float32; frames past an utterance's end are set to 0
 *              (the zero padding of model.py:135-141)
 * Frames per utterance: (n_samples - noverlap) / step if n_samples >= nperseg, else 0. */
int sb_log_specgram(const short* pcm, const long long* offsets, const int* n_samples, int B,
                    int nperseg, int step, double scale, float eps, const float* mean,
                    const float* stdev, float* out, int max_frames, void* stream);

/* Developer hook (not part of the drop-in surface): device buffer of >= 64*16 uint64 receiving a
 * globaltimer timeline of CTA 0 for the next sb_gru_fwd launches; NULL disables. */
int sb_debug_gru_timeline(void* dev_buffer);
/* Developer hook, GEMM kernel selection (0 = default, bits combine): 1 = run every sb_gemm_bf16_tn
 * with N > 64 on the 128 x 128 tiles of the one-CTA kernel instead of the 128 x 256 tiles over
 * 2-CTA clusters; 2 = the 2-CTA kernel stores its output straight from the registers instead of
 * through shared memory and TMA; 4 = the 2-CTA kernel writes no output at all (timing only). */
int sb_debug_gemm_flags(int flags);
/* Developer hook: which kernel the last sb_gemm_bf16_tn launched: "c2_128x256" (2-CTA clusters),
 * "128x128" / "128x64" / "128x32" (one CTA per tile at that tile shape), "none". */
const char* sb_debug_gemm_kernel(void);
/* Developer hook: how the last sb_gemm_bf16_tn wrote its output: "tma" / "tma_reduce" (2-CTA
 * kernel: tiles staged in shared memory, TMA bulk tensor stores / reduce-adds), "regs" (straight
 * from the registers), "skipped" (flag 4), "none" before the first launch. */
const char* sb_debug_gemm_epilogue(void);
/* Developer hook, GRU kernel selection / timing knobs (0 = defaults): 8 / 16 = never / always use
 * the transposed-accumulator K-split kernels, 32 = no K-split forward kernel, 64 / 128 = polling
 * mode of the grid barrier, 256 / 512 = always (wherever the K-split backward kernel applies) /
 * never use its L2 reduce-scatter mode (the mode the backward uses when both directions do not
 * fit as thread-block clusters but do fit without), 1024 = the K-split forward over 2-CTA clusters
 * wherever it applies (H % 128 == 0, at most 64 batch rows; by default only from H = 512 up),
 * 2048 = the wide kernels with no resident W_hh chunks wherever they apply (every width they
 * take, so that the weight stream is tested at small widths); 1 / 2 are timing ablations
 * (results become wrong). */
int sb_debug_gru_flags(int flags);
/* Developer hook: which forward recurrence kernel the last sb_gru_fwd launched: "plain", "kt"
 * (transposed-accumulator K split), "ks4" / "ks2" (K split over 4- / 2-CTA clusters), "wide"
 * (U units per CTA, W_hh partly streamed), "none". */
const char* sb_debug_gru_fwd_kernel(void);
/* Developer hook: which backward recurrence kernel the last sb_gru_bwd launched: "plain", "kt",
 * "ks4" (K split over 4-CTA clusters), "ks_l2" (its L2 reduce-scatter mode), "ks4_x2" (one
 * clustered launch per direction), "wide", "none". */
const char* sb_debug_gru_bwd_kernel(void);
/* Developer hook: plan of the last wide launch of a pass (backward = 0: sb_gru_fwd, 1: sb_gru_bwd):
 * out[0] = units per CTA, out[1] = resident and out[2] = streamed 64-wide K chunks of W_hh per
 * CTA; all three 0 when that launch ran another kernel. */
int sb_debug_gru_plan(int backward, int* out);
/* Developer hook: gather-ring size in KB of the wide recurrence kernels (kb > 0 sets it; returns the
 * size in use).  Changes the shared memory of the next wide plans and launches. */
int sb_debug_gru_wide_ring(int kb);
/* Developer hook: enable (1, default) / disable (0) the K-split backward GRU kernel. */
int sb_debug_gru_ksplit(int enable);
/* Developer hook: set the preferred thread-block-cluster size (1, 2, 4 or 8) of the GRU kernels;
 * returns the cluster size the last GRU launch actually used (0 = query only, -1 = bad value;
 * 1 after a launch without clusters, e.g. the L2 reduce-scatter mode). */
int sb_debug_gru_cluster(int cluster_size);

#ifdef __cplusplus
}
#endif
#endif /* SPEECH_B200_H_ */
