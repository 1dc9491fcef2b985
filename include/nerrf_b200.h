/* nerrf_b200 -- C-ABI of the H100-native NERRF AI hot path.
 *
 * The reference (Itz-Agasta/nerrf @ a38ae13) has NO FFI / plugin interface for this path
 * (SURVEY.md 8b): the ai/ module it names (README.md:72-76) was never written.  The entry
 * points below are therefore the boundary a maintainer WOULD bind from the Python `ai/`
 * package the README names; each cites the reference interface (prose) it realises.
 *
 * Conventions (SURVEY.md 8b):
 *   - plain pointers and sizes only; no torch / C++ types;
 *   - every entry point returns 0 on success, <0 on error; the message is available from
 *     nerrf_last_error() (thread-local); nothing throws across the ABI;
 *   - device-pointer entry points are asynchronous on `stream` (a cudaStream_t passed as
 *     void*; NULL = default stream), allocate nothing, and own nothing: the caller owns all
 *     inputs, outputs and workspaces;
 *   - *_host entry points take HOST pointers (pinned for async copies), do the H2D / D2H
 *     copies themselves and synchronise before returning; the only persistent allocations
 *     live inside an explicit opaque session handle (create / destroy).
 *   - all matrices row-major fp32; indices int32 (rowptr int32 or int64).
 */
#ifndef NERRF_B200_H
#define NERRF_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NERRF_ABI_VERSION 2   /* 2: guard arrays (planner spec v1), MCTS host session, nerrf_trace_path_flags */

#define NERRF_OK 0
#define NERRF_ERR_INVALID (-1)   /* bad argument (shape, alignment, unsupported size)      */
#define NERRF_ERR_CUDA (-2)      /* a CUDA runtime call / kernel launch failed              */
#define NERRF_ERR_NODEVICE (-3)  /* no sm_90 device                                         */
#define NERRF_ERR_WORKSPACE (-4) /* workspace too small                                     */

/* algo selector for the GraphSAGE-T layer */
#define NERRF_SAGE_ALGO_AUTO 0
#define NERRF_SAGE_ALGO_FFMA 1   /* fused gather+aggregate -> fp32 CUDA-core GEMM           */
#define NERRF_SAGE_ALGO_UMMA 2   /* fused gather+aggregate -> wgmma GEMM, 3-term bf16 split
                                    (6 MMAs per K step; fp32-equivalent accuracy)           */
#define NERRF_SAGE_ALGO_UMMA2 3  /* same with a 2-term split (3 MMAs; ~1e-5 relative)       */

/* OR into `algo` of nerrf_sage_layer_fwd_ex: long_ws already holds the hub-row scan of THIS graph and row
 * range (it depends on rowptr only), e.g. layers 2..L of one forward: skip the re-scan. */
#define NERRF_SAGE_FLAG_REUSE_LONG_SCAN 0x100
/* OR into `algo` (layer calls, nerrf_sage_forward, the host session): no L2 eviction-priority hints in the tensor-core
 * layer, every access at normal priority.  By default, at F = 64 / 128, its gathered source rows, self terms, output
 * rows and edge slices are loaded and stored evict-first.  The results are the same bits either way; the flag is there
 * to compare the two. */
#define NERRF_SAGE_FLAG_NO_L2_POLICY 0x200

typedef void* nerrf_stream_t;    /* cudaStream_t */

int nerrf_abi_version(void);
const char* nerrf_last_error(void);
/* sm count / compute capability of the current device; NERRF_ERR_NODEVICE if none. */
int nerrf_device_info(int* sm_count, int* cc_major, int* cc_minor);

/* ------------------------------------------------------------------ GraphSAGE-T (rows a1-a3)
 * Replaces: ai/models/GraphSAGE-T.py `GraphSAGE_T.forward` (README.md:73, ROADMAP.md:127;
 * behaviour: docs/content/docs/architecture.mdx:49-53,157, threat-model.mdx:176-189).
 * Graph = CSR by destination: rowptr[n_nodes+1], col[E] source ids, ew[E] temporal weights. */

/* K1 alone: m[r - row_begin] = sum_e ew_e * x[col_e] / max(sum_e ew_e, 1e-12) for rows
 * [row_begin,row_end).  F in {32, 64, 128}.  m is [(row_end-row_begin), F]. */
int nerrf_sage_aggregate(const float* x, const void* rowptr, int rowptr_is64, const int32_t* col,
                         const float* ew, float* m, int64_t n_nodes, int64_t row_begin,
                         int64_t row_end, int F, nerrf_stream_t stream);

/* One fused layer: out[v] = act([x_v || m_v] @ W + b) for v in [row_begin,row_end); out is the
 * FULL [n_nodes, H] array (rows outside the range untouched).  W [2F, H], b [H]; H == 128.
 * x, out, W, b (and node_w below) must be 16-byte aligned. */
int nerrf_sage_layer_fwd(const float* x, const void* rowptr, int rowptr_is64, const int32_t* col,
                         const float* ew, const float* W, const float* b, float* out,
                         int64_t n_nodes, int64_t row_begin, int64_t row_end, int F, int H,
                         int relu, int algo, nerrf_stream_t stream);

/* The same layer with the node head fused into its epilogue (used for the last layer):
 * additionally score[v] = sigmoid(out_v . node_w + node_b) for v in [row_begin,row_end). */
int nerrf_sage_layer_head_fwd(const float* x, const void* rowptr, int rowptr_is64, const int32_t* col,
                              const float* ew, const float* W, const float* b, float* out,
                              int64_t n_nodes, int64_t row_begin, int64_t row_end, int F, int H,
                              int relu, int algo, const float* node_w, float node_b, float* score,
                              nerrf_stream_t stream);

/* Full-option layer call.  node_w == NULL: no fused head.  long_ws (optional device scratch, size from
 * nerrf_sage_long_rows_workspace_bytes): destination rows with more than 128 in-edges ("hub" rows: popular files, process nodes) are
 * pre-aggregated chunk-wise by many CTAs into it instead of being gathered by a single warp; rows that do
 * not fit in the scratch (or long_ws == NULL) are processed inline -- same result, slower. */
int nerrf_sage_long_rows_workspace_bytes(int64_t n_edges, size_t* bytes);
int nerrf_sage_layer_fwd_ex(const float* x, const void* rowptr, int rowptr_is64, const int32_t* col,
                            const float* ew, const float* W, const float* b, float* out,
                            int64_t n_nodes, int64_t row_begin, int64_t row_end, int F, int H,
                            int relu, int algo, const float* node_w, float node_b, float* score,
                            void* long_ws, size_t long_ws_bytes, float* const* peer_out, int n_peers,
                            const uint8_t* peer_need, nerrf_stream_t stream);
/* peer_out (host array of n_peers <= 7 device pointers, or NULL): peer-mapped [n_nodes, H] buffers of the other
 * ranks of a 1-D sharded forward (CUDA IPC / symmetric memory over NVLink).  The layer's epilogue stores each
 * output row to `out` AND to every peer buffer: the per-layer embedding exchange is fused into the layer
 * kernel.  peer_need (device uint8 [n_nodes], or NULL): bit i set <=> peer_out[i]'s rank references that row as
 * a source, so only the rows a peer actually reads are sent to it.  n_peers == -1: peer_out[0] is an NVSwitch MULTICAST address of the buffer on all ranks (this one
 * included): each element is stored once with multimem.st and replicated by the switch.
 * The caller provides the cross-rank barrier between layers. */

/* Heads.  score[v] = sigmoid(h_v . node_w + node_b).  If edge_W != NULL also writes
 * proj[v] = (h_v.We[0:H,0], h_v.We[0:H,1], h_v.We[H:2H,0], h_v.We[H:2H,1])  (proj [n,4]). */
int nerrf_sage_node_head(const float* h, const float* node_w, float node_b, float* score,
                         const float* edge_W, float* proj, int64_t row_begin, int64_t row_end,
                         int H, nerrf_stream_t stream);
/* edge_logit[e] = proj[col_e][0:2] + proj[dst_e][2:4] + edge_b   (== [h_src||h_dst] @ We + be); col and edge_logit
 * may be NULL when the graph has no edges. */
int nerrf_sage_edge_head(const float* proj, const void* rowptr, int rowptr_is64, const int32_t* col,
                         const float* edge_b, float* edge_logit, int64_t row_begin,
                         int64_t row_end, nerrf_stream_t stream);

/* Whole forward on device pointers: L layers + node head.  W[l] is [2F_l, H], b[l] is [H]
 * (host arrays of device pointers).  h_out [n_nodes,H]; score_out [n_nodes]; workspace must
 * hold n_nodes*H floats when L > 1; any bytes beyond that (256-aligned) are used as the hub-row scratch
 * (see nerrf_sage_long_rows_workspace_bytes). */
int nerrf_sage_forward(const float* x, const void* rowptr, int rowptr_is64, const int32_t* col,
                       const float* ew, int64_t n_nodes, int f_in, int hidden, int num_layers,
                       const float* const* W, const float* const* b, const float* node_w,
                       float node_b, float* h_out, float* score_out, float* workspace,
                       size_t workspace_bytes, int algo, nerrf_stream_t stream);

/* ------------------------------------------------------------------ GraphSAGE-T layer backward (training; SURVEY.md 8f rank 3)
 * Replaces: the GraphSAGE-T half of ai/train.py "joint GNN+LSTM training script" (README.md:75; ROADMAP.md:62-69).
 * Given one layer's saved tensors -- input h_in [n,F], its aggregate m [n,F] (nerrf_sage_aggregate of h_in), output
 * y [n,H] -- and the gradient dy [n,H] of the loss w.r.t. y:
 *     dP = dy * [y > 0] (relu != 0) or dy;   db = sum_v dP[v];   dW = [h_in || m]^T dP  ([2F,H]);
 *     dZ = dP W^T;   dh = dZ[:, :F] + A^T dZ[:, F:]
 * A^T is a gather over the TRANSPOSED graph, CSR by source: t_rowptr [n+1], t_col [E] = destination of each out-edge,
 * t_w [E] = ew_e / max(weight sum of that destination, 1e-12).  dh == NULL skips the input gradient (first layer),
 * dW == NULL (with db) skips the weight gradient; t_col / t_w may be NULL when the graph has no edges.  fp32, no atomics,
 * the chunking of the dW reduction a function of n_nodes only: bit-reproducible on every card.  All pointers device,
 * 16-byte aligned; workspace from nerrf_sage_layer_bwd_workspace_bytes. */
int nerrf_sage_layer_bwd_workspace_bytes(int64_t n_nodes, int F, size_t* bytes);
int nerrf_sage_layer_bwd(const float* h_in, const float* m, const float* y, const float* dy, const float* W,
                         const void* t_rowptr, int t_rowptr_is64, const int32_t* t_col, const float* t_w,
                         float* dh, float* dW, float* db, float* workspace, size_t workspace_bytes,
                         int64_t n_nodes, int F, int H, int relu, nerrf_stream_t stream);

/* nerrf_sage_layer_bwd with the edge-weight gradient (node explanations, nerrf_b200.explain; DESIGN.md 1.1.1).  d_ew
 * [E] != NULL ACCUMULATES this layer's term of d(out)/d(ew) in CSR-by-destination order (rowptr [n+1], int32 or int64
 * when rowptr_is64; col, ew [E]: the graph the forward read):
 *     d_ew[e] += dZ[dst(e), F:] . (h_in[src(e)] - [S >= 1e-12] m[dst(e)]) / max(S, 1e-12),   S = sum of dst(e)'s weights
 * with S summed as nerrf_sage_aggregate sums it ([S >= 1e-12] is the gradient of torch's clamp_min) and h - m taken as
 * (h - r) - (m - r) against r = h_in of the row's first source (exactly 0 when a row's sources are one node).  One warp
 * per destination row, no atomics: bit-reproducible.  d_ew needs h_in and rowptr (col / ew / d_ew may be NULL when the
 * graph has no edges).  nerrf_sage_layer_bwd is this call with d_ew = NULL. */
int nerrf_sage_layer_bwd_ex(const float* h_in, const float* m, const float* y, const float* dy, const float* W,
                            const void* t_rowptr, int t_rowptr_is64, const int32_t* t_col, const float* t_w,
                            float* dh, float* dW, float* db, float* workspace, size_t workspace_bytes,
                            int64_t n_nodes, int F, int H, int relu, const void* rowptr, int rowptr_is64,
                            const int32_t* col, const float* ew, float* d_ew, nerrf_stream_t stream);

/* ------------------------------------------------------------------ node explanations (DESIGN.md 1.1.1)
 * Receptive-field extraction: for each of n_targets target nodes (int32 ids into a CSR-by-destination graph of n_nodes
 * nodes), its `hops`-hop in-neighbourhood: every node within distance <= hops - 1 keeps ALL its in-edges (in their
 * original order), nodes at distance hops keep none (their features only).  The result is one block-diagonal batched
 * CSR, the targets' blocks in target order, each block's nodes in ascending global id.
 *   _count: counts [2 * n_targets] = (nodes, edges) per target; (-1, -1) when its kept edges exceed max_edges.
 *   _fill:  for targets that fit (pass only those), with node_off / edge_off [n_targets] their blocks' first node / edge:
 *           out_rowptr [total nodes + 1] (int64), out_col [total edges] (int32, batched node ids), out_ew, out_epos (int64:
 *           the edge's CSR position in the input graph), out_node [total nodes] (global id of each batched node), out_x
 *           [total nodes, F_in] (the node features), out_target [n_targets] (each target's batched node id).
 * Deterministic (the output is a function of the graph and the targets).  workspace: nerrf_explain_subgraph_workspace_bytes,
 * max_edges in [0, 2^28); hops in 1..16.  All pointers device. */
int nerrf_explain_subgraph_workspace_bytes(int64_t n_targets, int64_t max_edges, size_t* bytes);
int nerrf_explain_subgraph_count(const void* rowptr, int rowptr_is64, const int32_t* col, int64_t n_nodes,
                                 const int32_t* targets, int64_t n_targets, int hops, int64_t max_edges,
                                 int64_t* counts, void* workspace, size_t workspace_bytes, nerrf_stream_t stream);
int nerrf_explain_subgraph_fill(const void* rowptr, int rowptr_is64, const int32_t* col, const float* ew,
                                const float* x, int F_in, int64_t n_nodes, const int32_t* targets, int64_t n_targets,
                                int hops, int64_t max_edges, const int64_t* node_off, const int64_t* edge_off,
                                int64_t* out_rowptr, int32_t* out_col, float* out_ew, int64_t* out_epos,
                                int32_t* out_node, float* out_x, int32_t* out_target, void* workspace,
                                size_t workspace_bytes, nerrf_stream_t stream);
/* Segmented top-k: per segment t (edges [seg[t], seg[t+1]) of a batched graph), the k edges of largest
 * |a_e| = |ew[e] * d_ew[e]|, ties to the lower index, in that order: out_edge [n_seg, k] (batched edge index, -1 past the
 * segment's end), out_attr (a_e), out_pos (epos[e], or e when epos is NULL) and, when out_event != NULL, out_event =
 * edge_event[out_pos] (-1 when edge_event is NULL or the pick is empty).  One CTA per segment, k in 1..1024. */
int nerrf_explain_topk(const int64_t* seg, int64_t n_seg, const float* ew, const float* d_ew, const int64_t* epos,
                       const int64_t* edge_event, int k, int64_t* out_edge, float* out_attr, int64_t* out_pos,
                       int64_t* out_event, nerrf_stream_t stream);
/* Sequence-step evidence of the BiLSTM (DESIGN.md 1.2.1): per sequence b (seq, dseq fp32 [B, T, D_in]; dseq = the
 * gradient of its encrypt logit, nerrf_lstm_input_grad), over the valid steps t < len[b] (len clamped to [0, T]):
 *     a_t = sum_d seq[b,t,d] * dseq[b,t,d]   (each product rounded, summed left to right, d ascending)
 * and the k steps of largest |a_t|, ties to the lower t, NaN below every number: out_step int32 [B, k] (t, -1 past the
 * valid steps), out_attr fp32 (a_t, 0 there), out_feature int32 (argmax_d |seq * dseq|, ties to the lower d, -1 when every
 * term is 0), out_event int64 (step_event[b, t] of int64 [B, T], -1 when step_event is NULL or the pick is empty).
 * One warp per sequence; k in 1..1024, D_in in 1..1024.  Deterministic.  All pointers device. */
int nerrf_lstm_explain_steps(const float* seq, const float* dseq, const int32_t* len, int64_t B, int T, int D_in,
                             const int64_t* step_event, int k, int32_t* out_step, float* out_attr, int32_t* out_feature,
                             int64_t* out_event, nerrf_stream_t stream);

/* ------------------------------------------------------------------ incidents (DESIGN.md 1.4)
 * Flagged files and their owners: F = {v : node_kind[v] == 0 and score[v] >= tau} plus the file nodes `seeds` (int64
 * [n_seeds], may repeat), in ascending node id -> out_files int32 [|F|].  Per flagged file f (row v = out_files[f] of the
 * CSR-by-destination graph, rowptr int32 or int64):
 *   owner o = the source of the last process in-edge of the row (edge_attack == NULL), or the process source with the
 *     highest edge_attack[e] (NaN above every number), ties to the later position; -1 when the row has no process source;
 *   first / last = the lowest / highest position of the row whose source is o (the row's first / last position when
 *     o = -1, -1 when the row is empty); later = the positions p > first whose source is a process other than o (0 when
 *     o = -1);
 *   out_int int64 [n_nodes, 6] rows (o, first, last, later, edge_event[first], edge_event[last]) and out_real float64
 *   [n_nodes, 2] rows (edge_time[first], edge_time[last]); events -1 and times NaN where the position is -1 or the array
 *   is NULL.  Only the first |F| rows are written.
 * The call waits for `stream` once, to return |F| in *n_flagged (host) and to report bad input as NERRF_ERR_INVALID:
 * node_kind values other than 0 / 1, seeds outside [0, n_nodes) or not file nodes, any col id (all rowptr[n_nodes] of them) outside [0, n_nodes), tau NaN.
 * One warp per flagged row.  workspace: nerrf_incident_files_workspace_bytes.  All pointers device except n_flagged. */
int nerrf_incident_files_workspace_bytes(int64_t n_nodes, size_t* bytes);
int nerrf_incident_files(const void* rowptr, int rowptr_is64, const int32_t* col, int64_t n_nodes, const int8_t* node_kind,
                         const float* score, float tau, const int64_t* seeds, int64_t n_seeds, const float* edge_attack,
                         const double* edge_time, const int64_t* edge_event, int32_t* out_files, int64_t* out_int,
                         double* out_real, int64_t* n_flagged, void* workspace, size_t workspace_bytes, nerrf_stream_t stream);
/* Incidents of the n_flagged files of nerrf_incident_files (files, file_int, file_real as it wrote them): one per key
 * (node_source[file] (NULL = 0), owner), owner -1 = the source's unattributed incident.  Per incident, ordered by
 * (onset, source, owner; NaN onsets after every number, owner -1 last): inc_int int64 [n_flagged, 7] rows (source, owner,
 * offset of its files in grouped_files, n_files, onset event, end event, sum of `later`) and inc_real float64
 * [n_flagged, 4] rows (onset = min file onset, ties to the lower node id; end = max file end, same ties; NaN times never
 * win; sum of size_mb[file] as float64; max of score[file], NaN ignored).  grouped_files int32 [n_flagged]: each
 * incident's files in ascending node id; file_incident int32 [n_flagged]: each flagged file's incident index;
 * *n_incidents (device int32): the count.  Per-incident reductions run in a fixed lane order without atomics: two runs
 * give the same bits.  Asynchronous; workspace: nerrf_incident_group_workspace_bytes.  All pointers device. */
int nerrf_incident_group_workspace_bytes(int64_t n_flagged, size_t* bytes);
int nerrf_incident_group(const int32_t* files, const int64_t* file_int, const double* file_real, int64_t n_flagged,
                         const int32_t* node_source, const float* size_mb, const float* score, int32_t* n_incidents,
                         int64_t* inc_int, double* inc_real, int32_t* grouped_files, int32_t* file_incident,
                         void* workspace, size_t workspace_bytes, nerrf_stream_t stream);

/* ------------------------------------------------------------------ contamination (DESIGN.md 1.5)
 * Time-respecting causal closure over a CSR-by-destination graph (rowptr int32 or int64, col, node_kind 0 file /
 * 1 process as nerrf_incident_files).  Edge p of row v with source u = col[p] is open when its flow byte edge_flow[p]
 * (bit 0 process -> file, bit 1 file -> process; nerrf_trace_flow_class) has the bit of the pair's direction and
 * edge_time[p] (float64) is not NaN.  Seeds: distinct node ids (int64 [n_seeds]) with a seed time (float64, not NaN,
 * -inf / +inf allowed) and a label (int32 >= 0).
 *   phase 1: T0 = seed time (+inf elsewhere); Jacobi rounds: the (t, position)-smallest open edge of a row with
 *            T[col[p]] <= t_p replaces T[v] when t_p < T[v]; at most max_hops rounds (-1: until a round changes nothing);
 *   phase 2: level 0 = the seeds with T = their seed time; level k + 1 = the unlevelled nodes with T < +inf and a tight
 *            in-edge (open, T[col[p]] <= t_p = T[v]) from a level-k node; pred = the lowest such position, label =
 *            label[col[pred]].
 * Outputs, over the levelled nodes in ascending node id (n_nodes capacity each): out_nodes int32, out_time float64 (T),
 * out_level int32, out_pred int64 (-1 at level 0), out_label int32; *n_tainted, *n_rounds (rounds run) and *n_levels
 * (non-empty levels) on the host; stage_ms (host double [4], may be NULL): the host-clock milliseconds of validation,
 * phase 1, phase 2 and compaction, each ending in a stream wait.  The call waits once after validation, once per round
 * and per level, and once after compaction.  Bad input
 * is NERRF_ERR_INVALID: col ids outside [0, n_nodes) (all rowptr[n_nodes] of them), node_kind other than 0 / 1, flow
 * bytes above 3, seed ids out of range or repeated, NaN seed times, negative labels, max_hops < -1.  Results are
 * functions of the inputs alone (no atomics on values): two runs give the same bits.
 * workspace: nerrf_taint_closure_workspace_bytes.  All pointers device except the counts and stage_ms. */
int nerrf_taint_closure_workspace_bytes(int64_t n_nodes, size_t* bytes);
int nerrf_taint_closure(const void* rowptr, int rowptr_is64, const int32_t* col, int64_t n_nodes, const int8_t* node_kind,
                        const uint8_t* edge_flow, const double* edge_time, const int64_t* seeds, const double* seed_time,
                        const int32_t* seed_label, int64_t n_seeds, int max_hops, int32_t* out_nodes, double* out_time,
                        int32_t* out_level, int64_t* out_pred, int32_t* out_label, int64_t* n_tainted, int32_t* n_rounds,
                        int32_t* n_levels, double* stage_ms, void* workspace, size_t workspace_bytes, nerrf_stream_t stream);
/* The flow class of every event (the table of DESIGN.md 1.5) from its raw event slot (uint8), open flags and return
 * value: nerrf_trace_flow_class takes host columns (flags int64), nerrf_trace_flow_class_device device columns (flags
 * int32, the live decoder's); both evaluate the same definition.  The device call is asynchronous. */
int nerrf_trace_flow_class(const uint8_t* event_slot, const int64_t* flags, const int64_t* ret_val, int64_t n, uint8_t* flow_out);
int nerrf_trace_flow_class_device(const uint8_t* event_slot, const int32_t* flags, const int64_t* ret_val, int64_t n,
                                  uint8_t* flow_out, nerrf_stream_t stream);

/* The normalised edge weights of the graph, for t_w above: a[e] = ew[e] * (1 / max(weight sum of e's destination row,
 * 1e-12)), edges in CSR-by-destination order (rowptr [n+1], int32 or int64 when rowptr_is64; ew, a [E]).  The weight sum
 * is taken in the order nerrf_sage_aggregate takes it, so the entries are the forward's to the bit.  No atomics:
 * bit-reproducible.  ew and a may be NULL when the graph has no edges. */
int nerrf_sage_norm_weights(const void* rowptr, int rowptr_is64, const float* ew, float* a, int64_t n_nodes,
                            nerrf_stream_t stream);

/* Edge head backward (training the attack / normal edge classifier).  Forward = nerrf_sage_node_head (proj) +
 * nerrf_sage_edge_head.  Given d_logit [E,2] = d loss / d edge_logit in CSR-by-destination order:
 *     g_src[v] = sum_{e: src(e)=v} d_logit[e],   g_dst[v] = sum_{e: dst(e)=v} d_logit[e]
 *     dh[v] = g_src[v] We[0:H]^T + g_dst[v] We[H:2H]^T    ([n,H])
 *     d_edge_W = [h^T g_src ; h^T g_dst]  ([2H,2]),   d_edge_b = sum_v g_dst[v]  ([2])
 * t_rowptr [n+1] / t_eid [E] is the transposed graph (CSR by source): t_eid[j] = CSR-by-destination position of the j-th
 * out-edge; both int32, or int64 when t_is64.  dh == NULL skips the input gradient, d_edge_W == NULL skips the weight and
 * bias gradients (and the workspace).  H must be 128; h, edge_W, d_logit, dh, d_edge_W and workspace 16-byte aligned;
 * workspace from nerrf_sage_edge_head_bwd_workspace_bytes.  fp32, no atomics, chunking a function of n_nodes only:
 * bit-reproducible. */
int nerrf_sage_edge_head_bwd_workspace_bytes(int64_t n_nodes, int H, size_t* bytes);
int nerrf_sage_edge_head_bwd(const float* h, const float* edge_W, const float* d_logit,
                             const void* rowptr, int rowptr_is64,
                             const void* t_rowptr, const void* t_eid, int t_is64,
                             float* dh, float* d_edge_W, float* d_edge_b,
                             void* workspace, size_t workspace_bytes,
                             int64_t n_nodes, int H, nerrf_stream_t stream);

/* Host-buffer session (the e2e call): device buffers live in the handle. */
typedef struct nerrf_sage_session nerrf_sage_session;
int nerrf_sage_session_create(int64_t max_nodes, int64_t max_edges, int f_in, int hidden,
                              int num_layers, nerrf_sage_session** out);
/* weights are HOST pointers: W[l] [2F_l,H], b[l] [H], node_w [H]; copied to the device once. */
int nerrf_sage_session_set_weights(nerrf_sage_session* s, const float* const* W,
                                   const float* const* b, const float* node_w, float node_b);
/* HOST in / HOST out: copies the graph + features H2D, runs forward, copies score (and h if
 * h_out_host != NULL) D2H, synchronises. */
int nerrf_sage_session_forward_host(nerrf_sage_session* s, const float* x_host,
                                    const int32_t* rowptr_host, const int32_t* col_host,
                                    const float* ew_host, int64_t n_nodes, int64_t n_edges,
                                    float* score_out_host, float* h_out_host, int algo);
/* Pipelined form of the same call (a stream of graphs, e.g. one per sliding-window tick): submit queues H2D -> forward ->
 * D2H on the session's streams and returns at once with a ticket; wait blocks until that ticket's outputs are in the
 * host buffers.  Two steps may be in flight (two device buffer sets): the upload of step i+1 overlaps the layers of
 * step i.  A third submit blocks until the oldest ticket is complete.  The host buffers of a ticket must stay valid and
 * unmodified until its wait returns.  forward_host == submit + wait. */
int nerrf_sage_session_submit_host(nerrf_sage_session* s, const float* x_host,
                                   const int32_t* rowptr_host, const int32_t* col_host,
                                   const float* ew_host, int64_t n_nodes, int64_t n_edges,
                                   float* score_out_host, float* h_out_host, int algo,
                                   uint64_t* ticket);
int nerrf_sage_session_wait(nerrf_sage_session* s, uint64_t ticket);
int nerrf_sage_session_destroy(nerrf_sage_session* s);

/* ------------------------------------------------------------------ rewards.score (row a6)
 * Replaces: ai/planner/rewards.py (README.md:74,115 `Reward = -(data_loss + 0.1*downtime)`;
 * threat-model.mdx:205-223).  states uint32 [B, n_words], n_words = 32*NW, NW = 1/2/4 for
 * A <= 1024/2048/4096; action a = bit (a&31) of word (a>>5).  Bit-exact fixed-order fp32.
 * guard (device int32 [A], or NULL): planner spec v1 -- guard[a] = index (0..31) of the "kill process" action
 * (threat-model.mdx:212-215) that makes reverting a durable, or -1; an applied action whose guard is NOT applied
 * additionally loses p_guard * p_a * size_a (the live process re-encrypts the file).  NULL = spec v0. */
int nerrf_reward_score(const uint32_t* states, int64_t B, const float* p, const float* size,
                       const float* cost, const int32_t* guard, int A, float* out, nerrf_stream_t stream);
/* Planner spec v2: cover (int32 [A], or NULL; device pointer here and in the device-pointer entry points below, host
 * pointer in the *_host_ex ones) -- cover[a] = index (0..31, < A) of the "restore from backup" action
 * (threat-model.mdx:216-219) of the directory that holds a's file, or -1.  An action that is not applied but whose cover
 * is applied is restored all the same: its data-loss term is (1-p_a)*size_a (plus the guard penalty while its guard is
 * not applied) and it adds no downtime.  cover[a] != a; a cover target is not covered itself and is not a guard target
 * (otherwise NERRF_ERR_INVALID).  The check reads `cover` and `guard` back to the host, so with a cover table a
 * device-pointer call synchronizes its stream before it launches.  Each *_ex entry point takes `cover` right after
 * `guard`; the plain symbols are the *_ex ones with cover = NULL (spec v1, bit for bit). */
int nerrf_reward_score_ex(const uint32_t* states, int64_t B, const float* p, const float* size,
                          const float* cost, const int32_t* guard, const int32_t* cover, int A, float* out,
                          nerrf_stream_t stream);

/* ------------------------------------------------------------------ planner.mcts.search (a5)
 * Replaces: ai/planner/mcts.py (README.md:74, ROADMAP.md:84; architecture.mdx:62-72).
 * Leaf-parallel UCT, one persistent cooperative kernel for all T iterations, ONE grid barrier per
 * iteration (every CTA keeps its own replica of the tree; DESIGN.md 2.2).
 * Workspace layout is private (it grows with the SM count); query its size first.  Outputs: root_n int32 [A_pad],
 * root_w fp32 [A_pad] (A_pad = 1024*NW), num_nodes int32 [1] -- all device pointers.
 * ln_table: device fp32 [T+2], ln_table[k] = fp32(ln(k*R)).  R must be a power of two. */
int nerrf_mcts_workspace_bytes(int A, int T, int R, size_t* bytes);
int nerrf_mcts_search(const float* p, const float* size, const float* cost, const int32_t* guard, int A,
                      const uint32_t* root_state, int R, int D, int T, uint64_t seed, float c,
                      float lo, float inv_range, const float* ln_table, int32_t* root_n,
                      float* root_w, int32_t* num_nodes, void* workspace, size_t workspace_bytes,
                      nerrf_stream_t stream);
int nerrf_mcts_search_ex(const float* p, const float* size, const float* cost, const int32_t* guard,
                         const int32_t* cover, int A, const uint32_t* root_state, int R, int D, int T, uint64_t seed,
                         float c, float lo, float inv_range, const float* ln_table, int32_t* root_n, float* root_w,
                         int32_t* num_nodes, void* workspace, size_t workspace_bytes, nerrf_stream_t stream);
/* HOST in / HOST out, one-shot (allocates + frees device memory internally, synchronous).
 * root_state_host and guard may be NULL. */
int nerrf_mcts_search_host(const float* p, const float* size, const float* cost, const int32_t* guard, int A,
                           const uint32_t* root_state_host, int R, int D, int T, uint64_t seed,
                           float c, float lo, float inv_range, const float* ln_table_host,
                           int32_t* root_n_host, float* root_w_host, int32_t* num_nodes_host);
int nerrf_mcts_search_host_ex(const float* p, const float* size, const float* cost, const int32_t* guard,
                              const int32_t* cover, int A, const uint32_t* root_state_host, int R, int D, int T,
                              uint64_t seed, float c, float lo, float inv_range, const float* ln_table_host,
                              int32_t* root_n_host, float* root_w_host, int32_t* num_nodes_host);
/* plan(): validate-and-commit loop on the device (architecture.mdx:81-86 "sandbox validates, then apply"; the commit half of
 * ai/planner/mcts.py plan()).  cand[n_cand] (device int32, ranked root children of a search) are scored as score(state + c)
 * with the exact reward; the highest-ranked improving one is committed, the candidates that still improved stay in the list;
 * repeated up to max_commits times.  allow_tentative != 0: if nothing improves at the first round the first candidate is
 * committed anyway (spec-v1 lookahead).  state (device uint32 [32*NW]) is updated in place; actions_out / scores_out
 * [max_commits] and n_out[2] = {commits made, candidates left} are device arrays.  Asynchronous on `stream`; one cooperative
 * launch.  Decisions and scores are bit-identical to doing the loop with nerrf_reward_score on the host. */
int nerrf_plan_commit_workspace_bytes(int n_cand_max, size_t* bytes);
int nerrf_plan_commit(const float* p, const float* size, const float* cost, const int32_t* guard, int A,
                      uint32_t* state, const int32_t* cand, int n_cand, float cur, int max_commits,
                      int allow_tentative, int32_t* actions_out, float* scores_out, int32_t* n_out,
                      void* workspace, size_t workspace_bytes, nerrf_stream_t stream);
int nerrf_plan_commit_ex(const float* p, const float* size, const float* cost, const int32_t* guard,
                         const int32_t* cover, int A, uint32_t* state, const int32_t* cand, int n_cand, float cur,
                         int max_commits, int allow_tentative, int32_t* actions_out, float* scores_out, int32_t* n_out,
                         void* workspace, size_t workspace_bytes, nerrf_stream_t stream);

/* HOST in / HOST out through a session: the device buffers and a stream live in the handle (create once for the
 * largest A / T / R; a search is then six small H2D copies, one launch and three D2H copies, no allocation).
 * A must have the same word count NW as A_max. */
typedef struct nerrf_mcts_session nerrf_mcts_session;
int nerrf_mcts_session_create(int A_max, int T_max, int R_max, nerrf_mcts_session** out);
int nerrf_mcts_session_search_host(nerrf_mcts_session* s, const float* p, const float* size, const float* cost,
                                   const int32_t* guard, int A, const uint32_t* root_state_host, int R, int D, int T,
                                   uint64_t seed, float c, float lo, float inv_range, const float* ln_table_host,
                                   int32_t* root_n_host, float* root_w_host, int32_t* num_nodes_host);
int nerrf_mcts_session_search_host_ex(nerrf_mcts_session* s, const float* p, const float* size, const float* cost,
                                      const int32_t* guard, const int32_t* cover, int A, const uint32_t* root_state_host,
                                      int R, int D, int T, uint64_t seed, float c, float lo, float inv_range,
                                      const float* ln_table_host, int32_t* root_n_host, float* root_w_host,
                                      int32_t* num_nodes_host);
int nerrf_mcts_session_destroy(nerrf_mcts_session* s);

/* ------------------------------------------------------------------ lstm.forward (row a4)
 * Replaces: ai/models/lstm.py (README.md:73; architecture.mdx:55-59; threat-model.mdx:191-203).
 * BiLSTM, torch.nn.LSTM gate order (i,f,g,o).  seq [B,T,D_in]; len int32 [B] (valid steps
 * t < len[b]).  Weights per layer l and direction d (index 2*l+d), PRE-TRANSPOSED by the host:
 *   Wih_t[2l+d] [D_l, 4H],  Whh_t[2l+d] [H, 4H],  bias[2l+d] [4H] (= b_ih + b_hh);
 * D_0 = D_in, D_l = 2H.  head_W [2, 2H], head_b [2].  out [B,2] = sigmoid(head).
 * workspace: 2 * B*T*2H floats (layer outputs ping-pong).  H must be 256; B any. */
int nerrf_lstm_workspace_bytes(int64_t B, int T, int H, size_t* bytes);
int nerrf_lstm_forward(const float* seq, const int32_t* len, int64_t B, int T, int D_in, int H,
                       int num_layers, const float* const* Wih_t, const float* const* Whh_t,
                       const float* const* bias, const float* head_W, const float* head_b,
                       float* out, void* workspace, size_t workspace_bytes,
                       nerrf_stream_t stream);

/* ------------------------------------------------------------------ BiLSTM training (forward with saved activations +
 * backward-through-time; the BiLSTM half of ai/train.py "joint GNN+LSTM training script", README.md:75)
 * nerrf_lstm_forward_train runs the fp32 CUDA-core recurrence of nerrf_lstm_forward (same arguments, same pre-transposed
 * weights, no head) and writes the top layer's final states hfin_out [B,2H] = [h_fwd_final || h_bwd_final] -- the
 * head's input -- plus a tape of every layer's output, gates and cell states (tape_bytes from
 * nerrf_lstm_train_workspace_bytes).  nerrf_lstm_backward differentiates sum(dhfin * hfin) through that tape:
 *     per step, in reverse direction order:  dc += dh*o*(1 - tanh^2 c);  pre-activation gate gradients dg from the saved
 *     gates and c_{t-1};  dh_{t-1} = dg W_hh + d out_l[t-1];  dc_{t-1} = dc*f   (padded steps pass dh, dc through)
 *     dW_ih = dg^T in_l,  dW_hh = dg^T h_{t-1},  db = sum dg,  d in_l = [dg_fwd || dg_bwd] [W_ih_fwd ; W_ih_bwd]
 * W_ih[2l+d] [4H,D_l], W_hh[2l+d] [4H,H] are in torch's layout (NOT transposed), and so are the gradients it writes:
 * dW_ih[2l+d], dW_hh[2l+d], db[2l+d] [4H] (db is the gradient of both b_ih and b_hh).  dseq [B,T,D_in] == NULL skips
 * the input gradient; it is exactly 0 at padded steps.  The backward overwrites the tape's gates, so a tape is
 * differentiated once.  fp32, no atomics: bit-reproducible.  H must be 256; all pointers device (the pointer arrays are
 * host arrays of 2*num_layers device pointers), tape and workspace 16-byte aligned.  Asynchronous on `stream`. */
int nerrf_lstm_train_workspace_bytes(int64_t B, int T, int D_in, int H, int num_layers, size_t* tape_bytes,
                                     size_t* workspace_bytes);
int nerrf_lstm_forward_train(const float* seq, const int32_t* len, int64_t B, int T, int D_in, int H,
                             int num_layers, const float* const* Wih_t, const float* const* Whh_t,
                             const float* const* bias, float* hfin_out, void* tape, size_t tape_bytes,
                             nerrf_stream_t stream);
int nerrf_lstm_backward(const float* seq, const int32_t* len, int64_t B, int T, int D_in, int H, int num_layers,
                        const float* const* W_ih, const float* const* W_hh, void* tape, size_t tape_bytes,
                        const float* dhfin, float* dseq, float* const* dW_ih, float* const* dW_hh, float* const* db,
                        void* workspace, size_t workspace_bytes, nerrf_stream_t stream);
/* Input gradient only (explanations, DESIGN.md 1.2.1): nerrf_lstm_backward without dW_ih, dW_hh and db.  It runs the same
 * recurrence and input-gradient launches and skips the weight gradients, so dseq (required here) equals
 * nerrf_lstm_backward's on the same tape bit for bit.  The workspace is the layer-output gradient buffer alone
 * (B*T*2H floats, rounded up to 256 bytes); tape_bytes as for nerrf_lstm_backward.  Consumes the tape the same way. */
int nerrf_lstm_input_grad_workspace_bytes(int64_t B, int T, int D_in, int H, int num_layers, size_t* bytes);
int nerrf_lstm_input_grad(const float* seq, const int32_t* len, int64_t B, int T, int D_in, int H, int num_layers,
                          const float* const* W_ih, const float* const* W_hh, void* tape, size_t tape_bytes,
                          const float* dhfin, float* dseq, void* workspace, size_t workspace_bytes, nerrf_stream_t stream);

/* ------------------------------------------------------------------ temporal-graph constructor, device half
 * (SURVEY.md 8f rank 1 -- the step immediately before GraphSAGE_T.forward)
 * Replaces: the graph-constructor stage the reference documents but does not ship
 * (docs/content/docs/architecture.mdx:32-42 sliding window, inode dedup, "edge weight = causality
 * confidence"; node schema :144-160; input records proto/trace.proto:11-49).
 * Edge list (device, int32 src/dst in [0, n_nodes), fp32 event time t and confidence conf) ->
 * CSR-by-destination in exactly the layout nerrf_sage_forward reads:
 *   edges stably sorted by (dst, t);  col[i] = src;  ew[i] = conf * exp(-(t_ref - t) / tau);
 *   rowptr[v] = #edges with dst < v   (int32, or int64 when rowptr_is64; n_edges >= 2^31 needs int64).
 * rowptr and col are bit-exact against the host constructor (nerrf_b200/graph.py csr_from_edges);
 * ew differs only by the exp implementation (<= 2 ulp).  Deterministic (no atomics).
 * Limits: n_edges < 2^32, n_nodes < 2^31.  workspace: nerrf_graph_csr_workspace_bytes, 256-byte
 * aligned.  The call waits for `stream` once, to report out-of-range vertex ids as NERRF_ERR_INVALID. */
int nerrf_graph_csr_workspace_bytes(int64_t n_edges, int64_t n_nodes, int64_t* bytes);
int nerrf_graph_build_csr(const int32_t* src, const int32_t* dst, const float* t, const float* conf,
                          int64_t n_edges, int64_t n_nodes, float t_ref, float tau,
                          void* rowptr_out, int rowptr_is64, int32_t* col_out, float* ew_out,
                          void* workspace, int64_t workspace_bytes, nerrf_stream_t stream);
/* The same, and also perm_out[i] (device uint32 [n_edges], may be NULL) = index in the INPUT edge list of the edge at CSR
 * position i -- lets later stages (the per-file event sequences) go back from a CSR row to the events that made it. */
int nerrf_graph_build_csr_ex(const int32_t* src, const int32_t* dst, const float* t, const float* conf,
                             int64_t n_edges, int64_t n_nodes, float t_ref, float tau, void* rowptr_out,
                             int rowptr_is64, int32_t* col_out, float* ew_out, uint32_t* perm_out, void* workspace,
                             int64_t workspace_bytes, void* stream);
/* Per-file event sequences for lstm.forward on the device (architecture.mdx:55-59 "last 100 events per file"; spec =
 * nerrf_b200/ingest.py sequences_core): for every candidate file node its last t_max events, oldest first, as
 * seq_out [n_cand, t_max, 16] fp32 (zero padded) + len_out [n_cand].  Graph built from the window's events in time order
 * with TWO edges per event (process -> file, file -> process: merge_renames mode), perm from nerrf_graph_build_csr_ex, order
 * [n_window] = stored index of the window's events by rank; ts / event_slot / bytes / path_flags are the stored columns.
 * All pointers device. */
int nerrf_trace_sequences(const int64_t* cand_nodes, int n_cand, const void* rowptr, int rowptr_is64, const uint32_t* perm,
                          const int64_t* order, const double* ts, const uint8_t* event_slot, const int64_t* bytes,
                          const uint8_t* path_flags, double t0, double span, int t_max, float* seq_out,
                          int32_t* len_out, void* stream);
/* The same, and also event_out (int64 [n_cand, t_max], may be NULL): event_out[c, k] = order[perm[e] >> 1], the stored
 * row of the event that made step k of candidate c (the id space of the stream's event records), -1 at padded steps.
 * The plain symbol is this call with event_out = NULL; seq_out and len_out are the same bits either way. */
int nerrf_trace_sequences_ex(const int64_t* cand_nodes, int n_cand, const void* rowptr, int rowptr_is64,
                             const uint32_t* perm, const int64_t* order, const double* ts, const uint8_t* event_slot,
                             const int64_t* bytes, const uint8_t* path_flags, double t0, double span, int t_max,
                             float* seq_out, int32_t* len_out, int64_t* event_out, void* stream);

/* Per-pair edge labels of a trace graph on the device (the training target of the edge head; spec = nerrf_b200/graph.py
 * graph_from_events meta['edge_label']).  node_p / node_f [n_events] = the graph's events mapped to node ids (as handed
 * to nerrf_graph_node_features), raw_slot [n_events] = their ANNOTATION event slots (not the observable fold);
 * rowptr / col = the graph's CSR by destination (n_edges = rowptr[n_nodes]).  label_out uint8 [n_edges], CSR order: 1 iff
 * one end of the edge is a process p, the other a file f, and p has an event of raw slot 1..3 (encrypt start, encrypt
 * complete, ransom note) on f; 0 elsewhere, file <-> file rename links included.  Event ids outside [0, n_nodes) match
 * nothing.  Sort + binary search: deterministic, no atomics, does not wait for `stream`.  All pointers device. */
int nerrf_trace_edge_labels_workspace_bytes(int64_t n_events, int64_t* bytes);
int nerrf_trace_edge_labels(const int32_t* node_p, const int32_t* node_f, const uint8_t* raw_slot, int64_t n_events,
                            const void* rowptr, int rowptr_is64, const int32_t* col, int64_t n_edges, int64_t n_nodes,
                            uint8_t* label_out, void* workspace, int64_t workspace_bytes, nerrf_stream_t stream);

/* Per-node features on the device (rest of SURVEY.md 8f rank 1): event columns already mapped to node
 * ids (nerrf_trace_intern, events in time order) -> x [n_nodes, 32] in the layout GraphSAGE_T.forward
 * reads (node schema docs/content/docs/architecture.mdx:144-160, threat-model.mdx:154-184; column
 * meaning nerrf_b200/graph.py graph_from_events): 0 file, 1 process, 3/4 log1p(in/out degree),
 * 5..12 log1p(event-kind counts), 13 log1p(bytes)/20, 14 (last-first)/window, 15 first/window,
 * 16 .lockbit, 17 ransom-note, 18 /tmp|/proc, 19 completes/(starts+writes); label_out (0/1: the file
 * was encrypted) and size_mb_out are optional.  Device pointers; t = seconds since the first event
 * (>= 0, double); node_g may be NULL (no rename targets).  Integer atomics only -> deterministic;
 * equals the host constructor up to the rounding of log1p (<= 1 ulp of fp32).  Waits for `stream`
 * once to report malformed columns. */
int nerrf_graph_node_features_workspace_bytes(int64_t n_nodes, int64_t* bytes);
int nerrf_graph_node_features(const int32_t* node_p, const int32_t* node_f, const int32_t* node_g,
                              const double* t, const uint8_t* event_slot, const uint64_t* bytes,
                              const uint8_t* path_flags, int64_t n_events, const int8_t* node_kind,
                              int64_t n_nodes, double window, float* x_out, int32_t* label_out,
                              float* size_mb_out, void* workspace, int64_t workspace_bytes,
                              nerrf_stream_t stream);

/* ------------------------------------------------------------------ EventBatch ingest (HOST code)
 * (SURVEY.md 8f rank 2 -- the wire format on the input side of the path)
 * Replaces: the consumer of the tracker's gRPC stream (proto/trace.proto:11-49 Event, :47-49
 * EventBatch; producer tracker/cmd/tracker/main.go:229-252).  `buf` holds one serialized
 * nerrf.trace.EventBatch, or any number of them concatenated (repeated fields append).
 * nerrf_trace_scan counts the events (top-level hop) and gives an upper bound per string column
 * (string_bytes[4] = comm, syscall, path, new_path; exact totals are off[n_events] after decoding);
 * nerrf_trace_decode parses the events once and fills caller-owned arrays: scalars [n_events]; strings as offsets [n_events+1]
 * + packed bytes; event_slot = graph feature slot of the syscall name (0 file_created,
 * 1 file_encrypt_start, 2 file_encrypt_complete, 3 ransom_note_created, 4 openat, 5 write,
 * 6 rename, 7 other); path_flags = NERRF_PATH_* bits of `path`.  Malformed input ->
 * NERRF_ERR_INVALID with the byte offset in nerrf_last_error().
 * Events must name a file: the tracker zeroes `path` on write events (tracker/bpf/tracepoints.c:62-64); the host
 * side (nerrf_b200/ingest.py resolve_columns) attributes those to the pid's last non-empty path before interning.
 * nerrf_trace_intern: pid / path interning ("merge by inode", architecture.mdx:41): node ids in
 * order of first appearance over events visited in `order` (NULL = as stored); node tables sized
 * by the caller (node_capacity >= 2*n_events with merge_renames, 3*n_events without); with merge_renames a
 * non-empty new_path aliases its merge key to the event's file node (a real rename a.dat -> a.dat.lockbit3);
 * node_name_which: 0 = path, 1 = new_path of event node_name_event, 2 = the pid itself. */
#define NERRF_PATH_LOCKBIT   1   /* ".lockbit" in path */
#define NERRF_PATH_NOTE      2   /* README / RANSOM (ASCII case-insensitive) in path */
#define NERRF_PATH_TMP       4   /* path starts with /tmp or /proc */
#define NERRF_PATH_ENCRYPTED 8   /* path ends with ".lockbit3" (benchmarks/m1/scripts/m1_rollback.sh:95) */
int nerrf_trace_scan(const uint8_t* buf, int64_t len, int64_t* n_events, int64_t* string_bytes);
int nerrf_trace_decode(const uint8_t* buf, int64_t len, int64_t n_events,
                       int64_t* ts_sec, int32_t* ts_nanos, uint32_t* pid, uint32_t* tid,
                       int32_t* flags, int64_t* ret_val, uint64_t* bytes,
                       uint8_t* event_slot, uint8_t* path_flags,
                       int64_t* comm_off, uint8_t* comm_data, int64_t* syscall_off, uint8_t* syscall_data,
                       int64_t* path_off, uint8_t* path_data, int64_t* new_path_off, uint8_t* new_path_data);
/* NERRF_PATH_* bits for every string of a packed string column (off [n+1], data): the rule nerrf_trace_decode
 * applies to `path`, available for `new_path` (a rename target names the file from then on). */
int nerrf_trace_path_flags(const int64_t* off, const uint8_t* data, int64_t n, uint8_t* flags_out);

/* Top-level framing of an EventBatch byte stream (HOST code), the walk of nerrf_trace_decode without parsing the
 * Events: for every Event record (field 1) rec_at = byte offset of its tag, body_off / body_len = its body; any other
 * top-level field is skipped by its wire type.  The first min(n, max_records) records are written and *n_records = n
 * (call again with a larger array when n > max_records).  *consumed = bytes covered by whole records.  partial != 0: a
 * trailing record that is merely cut off is left out of `consumed` (the caller carries it over to the next chunk);
 * partial == 0 or anything else malformed -> NERRF_ERR_INVALID, "malformed EventBatch at byte offset N", with the
 * outputs describing the records before N (an Event body is not checked here: nerrf_trace_decode_device does that). */
int nerrf_trace_frame(const uint8_t* buf, int64_t len, int partial, int64_t max_records, int64_t* rec_at,
                      int64_t* body_off, int64_t* body_len, int64_t* n_records, int64_t* consumed);

/* ------------------------------------------------------------------ live stream: EventBatch records decoded and
 * appended ON THE DEVICE (csrc/live_stream.cu; nerrf_b200/stream.py DeviceStream.live).
 * Columns are passed as a host array `cols` of 17 device pointers in the argument order of nerrf_trace_decode:
 * ts_sec, ts_nanos, pid, tid, flags, ret_val, bytes, event_slot, path_flags, comm_off, comm_data, syscall_off,
 * syscall_data, path_off, path_data, new_path_off, new_path_data.
 *
 * nerrf_trace_decode_device: the n_records records framed by nerrf_trace_frame (rec_at / body_off / body_len, device
 * copies; offsets into `buf`, the wire bytes on the device) are parsed by the host decoder's rules and written at rows
 * n_old .. n_old + n_records - 1; string offsets continue from off[n_old], so every data array needs room for
 * off[n_old] + the records' body bytes (which must stay below 2^31).  *status (device) = the smallest rec_at of a
 * malformed record, or all ones when every record parsed: the rows are only valid then.  Asynchronous on `stream`.
 * workspace: 256-byte aligned, nerrf_trace_decode_device_workspace_bytes. */
int nerrf_trace_decode_device_workspace_bytes(int64_t n_records, int64_t* bytes);
int nerrf_trace_decode_device(const uint8_t* buf, const int64_t* rec_at, const int64_t* body_off, const int64_t* body_len,
                              int64_t n_records, int64_t n_old, void* const* cols, uint64_t* status, void* workspace,
                              int64_t workspace_bytes, void* stream);
/* Time order, path resolution and retention of n_events resident events (device arrays):
 *   ts_out [n] = ts_sec + ts_nanos * 1e-9 in float64 (numpy's two roundings);
 *   src_out [n] = stored index of the event whose path the event uses: itself when its path is non-empty, else the pid's
 *     most recent event with a path in stable time order, or -1 (dropped) -- nerrf_b200/ingest.py resolve_columns;
 *   order_out [n_keep] = the surviving events in stable time order, ts_sorted_out [n_keep] their timestamps;
 *   res_path_off [n+1] = offsets of the resolved path column (dropped events: empty);
 *   retain_out [n_retain] (may be NULL) = in stored order, the events with ts > horizon and, per pid, its latest event
 *     with a path at or before the horizon (a later path-less write still resolves to it).
 * counts (HOST [3]) = n_keep, n_retain, total bytes of the resolved path column; the call synchronises the stream.
 * The resolved path column repeats a path for every path-less event that resolves to it, so it can be far larger than the
 * stored one: its size is summed in 64 bits, and 2^31 bytes or more is NERRF_ERR_INVALID (the offsets are scanned in
 * int32; the outputs are then unspecified and counts is zero).
 * workspace: 256-byte aligned, nerrf_trace_stream_order_workspace_bytes. */
int nerrf_trace_stream_order_workspace_bytes(int64_t n_events, int64_t* bytes);
int nerrf_trace_stream_order(int64_t n_events, const int64_t* ts_sec, const int32_t* ts_nanos, const uint32_t* pid,
                             const int64_t* path_off, double horizon, double* ts_out, int64_t* order_out,
                             double* ts_sorted_out, int64_t* src_out, int64_t* res_path_off, int64_t* retain_out,
                             int64_t* counts, void* workspace, int64_t workspace_bytes, void* stream);
/* The per-event columns the window graph reads, from src_out / res_path_off of nerrf_trace_stream_order: the resolved
 * path bytes (res_path_data), pf_raw_out = path_flags of the source event, pf_out = the same OR the NERRF_PATH_LOCKBIT bit
 * of new_path when merge_renames, slot_out = slot_map[event_slot] (slot_map: device uint8 [8], NULL = identity).
 * Asynchronous on `stream`. */
int nerrf_trace_stream_columns(int64_t n_events, const int64_t* src, const int64_t* path_off, const uint8_t* path_data,
                               const uint8_t* path_flags, const int64_t* new_path_off, const uint8_t* new_path_data,
                               const uint8_t* event_slot, const uint8_t* slot_map, const int64_t* res_path_off,
                               int merge_renames, uint8_t* res_path_data, uint8_t* pf_out, uint8_t* pf_raw_out,
                               uint8_t* slot_out, void* stream);
/* cols_out row k = cols_in row rows[k] (device int64 [n_rows], distinct rows, so every output data array fits in the
 * input's size); string offsets restart at 0.  The string bytes of the gathered rows, all four columns together, must
 * stay below 2^31 (one int32 scan turns their lengths into offsets; the call is asynchronous and cannot check the sum:
 * nerrf_b200/stream.py compact() does).  Asynchronous; workspace from nerrf_trace_gather_rows_workspace_bytes. */
int nerrf_trace_gather_rows_workspace_bytes(int64_t n_rows, int64_t* bytes);
int nerrf_trace_gather_rows(void* const* cols_in, const int64_t* rows, int64_t n_rows, void* const* cols_out,
                            void* workspace, int64_t workspace_bytes, void* stream);

/* The same interning ON THE DEVICE ("inode/path dedup via hash", SURVEY.md 8f rank 1; architecture.mdx:39-41): identical
 * nodes, numbering and names for the same events in the same processing order, computed by data-parallel passes (64-bit
 * hash + open-addressing table with first-mention atomicMin, rename-alias forest, creating-mention scan).  All array
 * arguments are DEVICE pointers; n_nodes is a HOST pointer (the call synchronises the stream).  The columns hold n_stored
 * events; the n_events events order[0..n_events) of them are processed in that order (order == NULL: the first n_events in
 * stored order) -- a sliding window over a resident stream is a slice of its time-sorted index array.  node_p / node_f /
 * node_g are written BY STORED INDEX (arrays of n_stored entries, only the processed events' entries are touched).  A 64-bit hash collision between two different keys is detected (keys are compared with their first mention's
 * bytes) and reported as an error, never merged silently.  workspace: 256-byte aligned, size from
 * nerrf_trace_intern_device_workspace_bytes. */
int nerrf_trace_intern_device_workspace_bytes(int64_t n_events, int64_t node_capacity, int64_t* bytes);
int nerrf_trace_intern_device(int64_t n_events, int64_t n_stored, const int64_t* order, const uint32_t* pid, const int64_t* path_off,
                              const uint8_t* path_data, const int64_t* new_path_off, const uint8_t* new_path_data,
                              int merge_renames, int32_t* node_p, int32_t* node_f, int32_t* node_g, int64_t* n_nodes,
                              int8_t* node_kind, int64_t* node_name_event, int8_t* node_name_which,
                              int64_t node_capacity, void* workspace, int64_t workspace_bytes, void* stream);
/* hash_out[v] = 64-bit hash of node v's NAME (the path / new_path of its naming event; pid nodes: the pid), device arrays:
 * lets a caller match nodes against a set of names without moving the strings (nerrf_b200/ingest.py name_hash is the same
 * function on the host). */
int nerrf_trace_name_hash(int64_t n_nodes, const int64_t* node_name_event, const int8_t* node_name_which,
                          const uint32_t* pid, const int64_t* path_off, const uint8_t* path_data,
                          const int64_t* new_path_off, const uint8_t* new_path_data, uint64_t* hash_out, void* stream);
/* The same hash over each node's parent DIRECTORY: the bytes of its name up to (not including) the last '/' (none: the
 * empty string); pid nodes hash as in nerrf_trace_name_hash.  Groups file nodes by directory for the planner's
 * "restore from backup" candidates.  Equals nerrf_b200/stream.py dir_hash bit for bit. */
int nerrf_trace_dir_hash(int64_t n_nodes, const int64_t* node_name_event, const int8_t* node_name_which,
                         const uint32_t* pid, const int64_t* path_off, const uint8_t* path_data,
                         const int64_t* new_path_off, const uint8_t* new_path_data, uint64_t* hash_out, void* stream);
int nerrf_trace_intern(int64_t n_events, const int64_t* order, const uint32_t* pid,
                       const int64_t* path_off, const uint8_t* path_data,
                       const int64_t* new_path_off, const uint8_t* new_path_data, int merge_renames,
                       int32_t* node_p, int32_t* node_f, int32_t* node_g, int64_t* n_nodes,
                       int8_t* node_kind, int64_t* node_name_event, int8_t* node_name_which,
                       int64_t node_capacity);

/* ------------------------------------------------------------------ several sources (one tracker per node)
 * Every event carries a source id s in [0, 2^16) (uint16 column, device or host like the other columns).  A process is
 * (s, pid) and a file is (s, path merge key): a rename target aliases within its own source, a path-less write resolves
 * to the latest named event of the same (s, pid), and retention keeps that event per (s, pid).  Name and directory
 * hashes are qualified by s and equal the unqualified ones at s = 0.  Each _ex entry point with source == NULL is the
 * entry point without the suffix, bit for bit (those are these calls with source = NULL).
 *
 * nerrf_trace_decode_device_ex: every decoded row gets source_col[row] = source (source_col NULL: not written).
 * nerrf_trace_stream_order_ex: key_bits 32 regroups by pid alone (4 radix passes; right whenever all events share one
 *   source), 48 by (source << 32) | pid (6 passes; needs the source column).
 * nerrf_trace_gather_rows_ex: also source_out[k] = source_in[rows[k]] (source_in NULL: 0; source_out NULL: skipped). */
int nerrf_trace_decode_device_ex(const uint8_t* buf, const int64_t* rec_at, const int64_t* body_off, const int64_t* body_len,
                                 int64_t n_records, int64_t n_old, void* const* cols, uint16_t* source_col, int source,
                                 uint64_t* status, void* workspace, int64_t workspace_bytes, void* stream);
int nerrf_trace_stream_order_ex(int64_t n_events, const int64_t* ts_sec, const int32_t* ts_nanos, const uint32_t* pid,
                                const uint16_t* source, int key_bits, const int64_t* path_off, double horizon,
                                double* ts_out, int64_t* order_out, double* ts_sorted_out, int64_t* src_out,
                                int64_t* res_path_off, int64_t* retain_out, int64_t* counts, void* workspace,
                                int64_t workspace_bytes, void* stream);
int nerrf_trace_gather_rows_ex(void* const* cols_in, const uint16_t* source_in, const int64_t* rows, int64_t n_rows,
                               void* const* cols_out, uint16_t* source_out, void* workspace, int64_t workspace_bytes,
                               void* stream);
int nerrf_trace_intern_device_ex(int64_t n_events, int64_t n_stored, const int64_t* order, const uint32_t* pid,
                                 const uint16_t* source, const int64_t* path_off, const uint8_t* path_data,
                                 const int64_t* new_path_off, const uint8_t* new_path_data, int merge_renames,
                                 int32_t* node_p, int32_t* node_f, int32_t* node_g, int64_t* n_nodes, int8_t* node_kind,
                                 int64_t* node_name_event, int8_t* node_name_which, int64_t node_capacity,
                                 void* workspace, int64_t workspace_bytes, void* stream);
int nerrf_trace_name_hash_ex(int64_t n_nodes, const int64_t* node_name_event, const int8_t* node_name_which,
                             const uint32_t* pid, const uint16_t* source, const int64_t* path_off, const uint8_t* path_data,
                             const int64_t* new_path_off, const uint8_t* new_path_data, uint64_t* hash_out, void* stream);
int nerrf_trace_dir_hash_ex(int64_t n_nodes, const int64_t* node_name_event, const int8_t* node_name_which,
                            const uint32_t* pid, const uint16_t* source, const int64_t* path_off, const uint8_t* path_data,
                            const int64_t* new_path_off, const uint8_t* new_path_data, uint64_t* hash_out, void* stream);
int nerrf_trace_intern_ex(int64_t n_events, const int64_t* order, const uint32_t* pid, const uint16_t* source,
                          const int64_t* path_off, const uint8_t* path_data, const int64_t* new_path_off,
                          const uint8_t* new_path_data, int merge_renames, int32_t* node_p, int32_t* node_f,
                          int32_t* node_g, int64_t* n_nodes, int8_t* node_kind, int64_t* node_name_event,
                          int8_t* node_name_which, int64_t node_capacity);

#ifdef __cplusplus
}
#endif
#endif /* NERRF_B200_H */
