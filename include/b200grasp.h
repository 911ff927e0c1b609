/*
 * b200grasp.h -- C ABI of the H100-native SAC learner (libb200grasp.so).
 *
 * Drop-in boundary for the ONE hot path of BarisYazici/deep-rl-grasping: the replay-buffer
 * minibatch gradient step that the reference delegates to stable_baselines.SAC (TF1) --
 *   constructed at  manipulation_main/training/sb_helper.py:104-128
 *   driven from     manipulation_main/training/sb_helper.py:175   (model.learn -> SAC._train_step)
 *   queried from    manipulation_main/utils.py:71                 (agent.predict)
 *   (de)serialised  manipulation_main/training/sb_helper.py:228-247, train_stable_baselines.py:95-104
 *
 * Conventions: every function returns 0 on success or a negative B2G_E* code and never throws
 * across the ABI; b2g_last_error() gives the message for the calling thread's last failure.  A
 * handle is single-owner and not thread-safe; it owns one CUDA stream and all of its device
 * memory.  Host arrays passed in are caller-owned and copied before the call returns (or, for the
 * *_async calls, before the next b2g_sync).  All floating point data is IEEE fp32 unless noted.
 * Parameter tensors use the TF variable names and layouts of the shipped SB zips (conv filters
 * HWIO, conv bias (1,n,1,1), dense kernels [in,out]) so get/set round-trips with them.
 */
#ifndef B200GRASP_H_
#define B200GRASP_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2G_OK 0
#define B2G_EINVAL (-1)   /* bad argument / unknown variable name / size mismatch            */
#define B2G_ECUDA (-2)    /* CUDA runtime error (no device, launch failure, out of memory)   */
#define B2G_ESTATE (-3)   /* call not valid in this state (e.g. sampling from an empty buffer) */
#define B2G_ENCCL (-4)    /* NCCL unavailable or failed                                      */

/* precision modes of the dense contractions (convs, cnn_fc1, fc0 layers) */
#define B2G_PREC_FP32_SIMT 0   /* fp32 FFMA on CUDA cores: bit-faithful fp32 arithmetic            */
#define B2G_PREC_BF16X3 1      /* wgmma BF16 hi/lo split, 3 MMAs, fp32 accumulate (~2^-16)        */
#define B2G_PREC_BF16 2        /* wgmma single-pass BF16 (fast mode; tolerance reported)           */

typedef struct b2g_sac b2g_sac;

/* Replaces the keyword arguments of sb.SAC(policy, env, policy_kwargs, gamma, buffer_size,
 * batch_size, learning_rate, ...) -- sb_helper.py:120-128 -- plus the shapes the policy class
 * would read from env.observation_space / action_space (robot.py:207-228). */
typedef struct b2g_sac_cfg {
  int32_t obs_h, obs_w, obs_c; /* CNN policy: NHWC obs, obs_c = image channels + 1 feature plane
                                  (custom_obs_policy.py:28-32).  obs_h == 0 selects the MLP policy */
  int32_t obs_dim;             /* MLP policy: flat observation size (101 for the encoder config)   */
  int32_t n_act;               /* 5 (actuator.py:72-73); <= 8                                      */
  int32_t hidden;              /* SAC.layers = [hidden, hidden]: 64 (config/gripper_grasp.yaml:81), 128, 192 or 256; else B2G_EINVAL */
  int32_t batch;               /* per-rank minibatch size                                          */
  int64_t buffer_capacity;     /* replay slots on this rank (config/gripper_grasp.yaml:82)         */
  float gamma, tau, target_entropy;
  uint64_t seed;               /* replay-index and policy-noise streams                            */
  int32_t precision;           /* B2G_PREC_*                                                       */
  int32_t device;              /* CUDA ordinal                                                     */
  int32_t rank, nranks;        /* data-parallel group; nranks == 1 -> no collective                */
  const void* nccl_id;         /* 128-byte ncclUniqueId shared by all ranks (nranks > 1)           */
  const char* nccl_lib;        /* optional path of libnccl.so.2 to dlopen; NULL = default search   */
} b2g_sac_cfg;

/* What SAC._train_step returns / logs (logs.csv columns policy_loss, qf1_loss, qf2_loss,
 * value_loss, entropy, ent_coef, ent_coef_loss) plus the parity scalars north_star names. */
typedef struct b2g_sac_metrics {
  float policy_loss, qf1_loss, qf2_loss, value_loss, ent_coef_loss, entropy, ent_coef;
  float grad_norm_pi, grad_norm_values, grad_ent;
  float mean_q1, mean_q2, mean_v, mean_logp;
  int64_t n_updates;
} b2g_sac_metrics;

const char* b2g_last_error(void);
int b2g_version(void);
/* writes a fresh 128-byte ncclUniqueId (rank 0 calls this, then shares it out of band) */
int b2g_nccl_unique_id(void* out128, const char* nccl_lib);

/* Replay storage.  The replay keeps a pool of frame_capacity observation frames; a transition references the frame of its obs
 * and of its next_obs.  b2g_replay_add stores every next_obs as a new frame, and row i's obs shares the frame of row i's next_obs
 * of the previous call when the two are bitwise equal (the learn loop's next_obs(t) == obs(t+1) within an episode), so
 * episodic streams need about cap * (1 + episode ends / transitions) + n_envs frames.  When a new frame would overwrite one a
 * live transition still references, the oldest transitions are dropped early (b2g_replay_info counts them) and sampling stays
 * uniform over the live ones.
 * u8_plane_mask: bit c declares image channel c (CNN policy, c < obs_c - 1; c < obs_c under B2G_CNN_NATURE) an 8-bit plane, stored as one byte per pixel;
 * b2g_replay_add then refuses (B2G_EINVAL, nothing stored) any value there that is not an integer in [0, 255].
 * NULL (the default) = frame_capacity 2 * buffer_capacity and no 8-bit planes.  From 2 * buffer_capacity frames on, every
 * transition keeps two frames of its own (sharing would save nothing): the bytes of two rows per transition, and nothing is
 * ever dropped early. */
typedef struct b2g_replay_cfg {
  int64_t frame_capacity;      /* >= buffer_capacity + 1 */
  uint32_t u8_plane_mask;
} b2g_replay_cfg;

/* The CNN policy's feature extractor.
 * B2G_CNN_AUGMENTED: create_augmented_nature_cnn(1) (custom_obs_policy.py): conv1 reads the first obs_c - 1 planes, pixel
 *   [0,0] of the last plane is one direct feature, 513 features; tensors model/pi/cnn1/w .. cnn_fc1/b.
 * B2G_CNN_NATURE: stable-baselines' plain nature_cnn (common/policies.py), the simplified environment's CnnPolicy: conv1 reads
 *   all obs_c planes (1 .. 8), no direct feature, 512 features; tensors model/pi/c1/w, c1/b, c2/w, c2/b, c3/w, c3/b, fc1/w (1024,512), fc1/b.
 *   u8_plane_mask may name any plane below obs_c.  The 4-float tail of a compact replay row is zero. */
enum { B2G_CNN_AUGMENTED = 0, B2G_CNN_NATURE = 1 };
typedef struct b2g_sac_net_cfg {
  int32_t extractor;           /* B2G_CNN_AUGMENTED or B2G_CNN_NATURE (CNN policy only: obs_h > 0)  */
} b2g_sac_net_cfg;

int b2g_sac_create(const b2g_sac_cfg* cfg, b2g_sac** out);   /* = b2g_sac_create2(cfg, NULL, out) */
int b2g_sac_create2(const b2g_sac_cfg* cfg, const b2g_replay_cfg* replay /* NULL = default */, b2g_sac** out);   /* = create3(.., NULL, ..) */
/* net == NULL: B2G_CNN_AUGMENTED.  B2G_CNN_NATURE with the MLP policy (obs_h == 0), or an unknown extractor: B2G_EINVAL.
 * A training-state file records the extractor: b2g_sac_state_load refuses a file of the other extractor. */
int b2g_sac_create3(const b2g_sac_cfg* cfg, const b2g_replay_cfg* replay, const b2g_sac_net_cfg* net, b2g_sac** out);
int b2g_sac_destroy(b2g_sac* h);
/* Peer-memory data parallelism (nranks > 1, one process per GPU of one NVLink node).  Every rank exports B2G_DP_EXPORT_BYTES
 * (CUDA IPC handles of its parameter arena, gradient receive arena and exchange block), the caller gathers the nranks blobs in rank
 * order (any out-of-band channel: the Python layer uses torch.distributed) and hands the concatenation to every rank.
 * From then on the optimiser launch of each gradient step is the collective: reduce-scatter of the gradients through peer
 * stores, Adam / Polyak on the owned slice, all-gather of the new parameters through peer stores -- no NCCL call on the path.
 * Replaces the all-reduce the reference's data-parallel wrapper would issue (reference: none -- SB 2.10 SAC is single-process;
 * SURVEY.md section 8e defines the N > 1 semantics this implements). */
#define B2G_DP_EXPORT_BYTES 192
int b2g_sac_dp_export(b2g_sac* h, void* out192);
int b2g_sac_dp_connect(b2g_sac* h, const void* all_exports /* nranks x B2G_DP_EXPORT_BYTES, rank order */, int nranks);
int b2g_debug_dp_stamps(b2g_sac* h, long long* out5);
/* host-only: [n][hw][cfull] observations -> compact replay rows [n][hw*(cfull-1)+4] (image planes | actuator value | 3 x 0), the layout
 * b2g_replay_add / b2g_sac_step_host_pipelined store and copy; needs no device */
int b2g_debug_compact_host(const float* src, float* dst, int n, int hw, int cfull, int threads);   /* bring-up: %globaltimer at the phase boundaries of the last launch */
int b2g_sync(b2g_sac* h);

/* ---- parameters: SB-zip variable names without the ":0" suffix (get_parameters / load_parameters,
 *      sb_helper.py:114-115) */
int b2g_param_count(const b2g_sac* h);
int b2g_param_info(const b2g_sac* h, int idx, const char** name, int64_t* numel, int32_t* ndim, int64_t shape[4]);
int b2g_get_param(b2g_sac* h, const char* name, float* dst, size_t numel);
int b2g_set_param(b2g_sac* h, const char* name, const float* src, size_t numel);
int b2g_get_grad(b2g_sac* h, const char* name, float* dst, size_t numel); /* gradient of the last step */
int b2g_get_adam(b2g_sac* h, const char* name, float* m, float* v, size_t numel);
int b2g_reset_optimizer(b2g_sac* h);   /* zero Adam moments and step counters (fresh tf.Session) */

/* ---- replay buffer (ReplayBuffer.add; stores UN-normalised obs/reward as SB does when a
 *      VecNormalize wraps the env) and VecNormalize statistics used at sample time
 *      (sb_helper.py:118-119; float64 like numpy) */
/* n rows of full observations (host or device memory).  With frame_capacity < 2 * buffer_capacity, 2 n <= frame_capacity;
 * otherwise a call larger than the ring keeps its last buffer_capacity rows, like any ring. */
int b2g_replay_add(b2g_sac* h, const float* obs, const float* act, const float* rew, const float* next_obs,
                   const float* done, int64_t n);
int64_t b2g_replay_size(const b2g_sac* h);
/* ReplayBuffer.storage[slot] ([SB2] common/buffers.py): one stored (raw) transition back to the host; any output may be
 * NULL.  slot must be live: one of the b2g_replay_size slots starting at the oldest transition (slot 0 unless transitions
 * were dropped early).  CNN policy: frames hold compact rows (see b2g_debug_compact_host), so obs and next_obs come back with
 * the image planes as stored and the actuator plane zero except pixel [0,0], the one value the policy reads of it. */
int b2g_replay_get(b2g_sac* h, int64_t slot, float* obs, float* act, float* rew, float* next_obs, float* done);
/* replay counters; any output may be NULL.  live_frames = frames from the oldest one a live transition references to the newest;
 * bytes = device memory of the replay (frames, frame indices, actions, rewards, dones) */
int b2g_replay_info(const b2g_sac* h, int64_t* capacity, int64_t* size, int64_t* frame_capacity, int64_t* live_frames,
                    int64_t* bytes, int64_t* evicted_early);
/* What the LAST gradient step (any entry point, the CUDA-graph path included) drew and produced: the replay slots
 * indices[batch] (sampled steps only), the policy noise eps[batch, n_act], the per-sample rows q1,q2,v,logp,v_targ,
 * q1_pi,q2_pi (7 x [batch]) and the squashed actions pi[batch, n_act].  Any pointer may be NULL.  This is what lets a
 * test replay the very batch of a sampled step in the oracle. */
int b2g_get_last_batch(b2g_sac* h, int32_t* indices, float* eps, float* per_sample, float* pi_out);
/* On a handle that owns obs_rms (b2g_obs_rms_set, below) obs_mean / obs_var may be NULL with norm_obs != 0: the scalars are
 * set and the device statistics stay; passing them replaces the device statistics (count kept). */
int b2g_set_norm_stats(b2g_sac* h, const double* obs_mean, const double* obs_var, double ret_var, double clip_obs,
                       double clip_rew, double eps, int norm_obs, int norm_reward);

/* ---- VecNormalize's observation statistics on the device, and the actor side of the learn loop fed from one upload per
 *      frame.  obs_rms = (mean[E], var[E], count), float64, E = H*W*C (or obs_dim) in the caller's observation layout: the
 *      RunningMeanStd that [SB2] VecNormalize keeps on the host.  b2g_obs_rms_set creates it on the handle (nranks == 1 only:
 *      each rank would own different statistics); from then on the table that the gather of the gradient step and policy
 *      inference normalise with is derived from it on the device, in the kernel that merges new frames, on the handle's
 *      stream: a step sampled after an observe call uses the statistics that call left, with no host round trip.
 *      Merge rule (RunningMeanStd.update_from_moments): per element, bm = mean and bv = biased variance of the n frames,
 *      summed in frame order 0 .. n-1; delta = bm - mean; tot = count + n; mean += delta * n / tot;
 *      var = (var * count + bv * n + delta^2 * count * n / tot) / tot; count = tot.
 *      Which frames are merged is VecNormalize's rule: reset() merges the reset frames (observe_act with obs), step_wait()
 *      merges the n frames the VecEnv returned -- for a finished env the frame its auto-reset returned, NOT the terminal
 *      observation, which goes into the replay only (observe_add).  With 8-bit replay planes the statistics are taken from the
 *      float frames as uploaded; a value there that is not an integer in [0, 255] is refused (B2G_EINVAL, nothing changed).
 *      Up to max(batch, 256) frames per call.  Like b2g_replay_add and b2g_sac_act, a call returns once the handle's stream
 *      has run what it enqueued. */
/* n raw observations (host, caller-owned, copied before return), or obs == NULL to act on the observations already staged.
 * update_stats != 0: merge them into the device obs_rms first (VecNormalize.training; B2G_ESTATE without b2g_obs_rms_set).
 * Then normalise with the CURRENT statistics, run the actor and write n actions; act_out == NULL skips the actor (a step
 * that explores with random actions).  The frames stay staged in the handle as "the current observation of env i". */
int b2g_sac_observe_act(b2g_sac* h, const float* obs, int n, int update_stats, int deterministic, float* act_out);
/* Transition i = (staged obs_i, act_i, rew_i, next_obs_i, done_i).  next_obs is uploaded ONCE: it goes into the replay as this
 * transition's next frame, is merged into obs_rms when update_stats != 0, and becomes the staged observation of env i unless
 * done_i, in which case reset_obs_i (the frame the auto-reset returned; merged instead, and the only rows of reset_obs that
 * are read) does.  With a frame-sharing replay the staged frame is linked, not stored again.  B2G_ESTATE before any
 * b2g_sac_observe_act; n must equal the number of staged observations. */
int b2g_sac_observe_add(b2g_sac* h, const float* act, const float* rew, const float* next_obs, const float* done,
                        const float* reset_obs /* may be NULL when no env finished */, int n, int update_stats);
/* obs_rms in and out (vecnormalize.pkl, sync_envs_normalization, resume): float64 [H*W*C] each + count.  set refuses a
 * negative or non-finite count, a negative variance and non-finite values (B2G_EINVAL); get returns B2G_ESTATE on a handle
 * without statistics; any output may be NULL. */
int b2g_obs_rms_set(b2g_sac* h, const double* mean, const double* var, double count);
int b2g_obs_rms_get(b2g_sac* h, double* mean, double* var, double* count);
/* bytes copied host -> device so far by b2g_sac_observe_* and b2g_obs_rms_set (observe_bytes) and by b2g_sac_act,
 * b2g_replay_add and b2g_set_norm_stats (other_bytes); either may be NULL */
int b2g_upload_bytes(const b2g_sac* h, int64_t* observe_bytes, int64_t* other_bytes);

/* ---- the hot path.  One call = n_steps x { sample -> normalise -> fwd -> bwd -> [allreduce] ->
 *      3x Adam -> Polyak }  (SAC._train_step + target_update_op).  Indices and policy noise come
 *      from the handle's counter-based generators.  metrics (may be NULL) = last step. */
int b2g_sac_step(b2g_sac* h, int n_steps, float lr, b2g_sac_metrics* out);
/* Same, but metrics stay on the device until b2g_sync/next blocking call (no host round trip). */
int b2g_sac_step_async(b2g_sac* h, int n_steps, float lr);

/* Parity entry point: the caller supplies the RAW batch (host pointers; normalised on the device
 * with the current statistics) and the N(0,1) noise eps[batch, n_act], so results are comparable
 * with the oracle.  per_sample (may be NULL) receives q1,q2,v,logp,v_targ,q1_pi,q2_pi as 7 rows of
 * [batch]; pi_out (may be NULL) receives tanh-squashed actions [batch, n_act].
 * apply_update == 0 computes losses and gradients only. */
int b2g_sac_step_explicit(b2g_sac* h, const float* obs, const float* act, const float* rew, const float* next_obs,
                          const float* done, const float* eps, float lr, int apply_update, b2g_sac_metrics* out,
                          float* per_sample, float* pi_out);

/* Same work as b2g_sac_step_explicit(apply_update = 1) for a caller that keeps its replay buffer on the HOST
 * (as stable-baselines does): the step is enqueued and the call returns the losses of the PREVIOUSLY enqueued step
 * (*have_prev = 0 on the first call), so the host->device copy of step k overlaps the compute of step k-1.  The
 * host arrays must stay valid until the next call or b2g_sac_pipeline_flush (use pinned memory for true overlap). */
int b2g_sac_step_host_pipelined(b2g_sac* h, const float* obs, const float* act, const float* rew, const float* next_obs,
                                const float* done, const float* eps, float lr, b2g_sac_metrics* prev_out, int* have_prev);
/* waits for the last pipelined step and returns its losses */
int b2g_sac_pipeline_flush(b2g_sac* h, b2g_sac_metrics* last_out);

/* policy_tf.step (SAC.predict, utils.py:71): obs are RAW, normalised with the current stats.
 * deterministic -> tanh(mu); else tanh(mu + eps*std) with eps from the handle's generator. */
int b2g_sac_act(b2g_sac* h, const float* obs, int n, int deterministic, float* act_out);

/* ---- training state: stop a run and continue it later.  The file holds what decides the next step / act / replay_add: the
 *      parameter arena (target network and log_ent_coef included), both Adam moments, the device counters (Adam steps,
 *      n_updates, the Philox step of the slot and noise draws, replay size and first live slot), the replay bookkeeping, the
 *      transition arrays and the live window of replay frames, and the device obs_rms of a handle that owns one.  Not in it: the
 *      other normalisation statistics (set them again with b2g_set_norm_stats; VecNormalize keeps its own file), the staged
 *      observations of b2g_sac_observe_* (a resumed run starts a fresh episode) and the precision mode (a bf16x3 state loads
 *      into an fp32 handle).
 * save: waits for every step enqueued on the handle; B2G_ESTATE while a host-pipelined step awaits b2g_sac_pipeline_flush and
 *       for nranks > 1 (data-parallel checkpoints are not built).
 * load: into a handle created with the same configuration.  The header, the configuration fingerprint (shape, n_act, hidden,
 *       batch, capacities, 8-bit planes, gamma, tau, target_entropy, seed, and whether obs_rms is carried: a file written with
 *       it loads only into a handle that owns one, and the reverse), the section lengths and the file size are checked
 *       before anything is written: a mismatch returns B2G_EINVAL naming the first field that differs and leaves the handle as
 *       it was.  A read or checksum failure after that leaves the handle unusable: every call but destroy and another load
 *       then returns B2G_ESTATE. */
int b2g_sac_state_save(b2g_sac* h, const char* path);
int b2g_sac_state_load(b2g_sac* h, const char* path);

/* ---- per-step metrics log (TensorBoard).  With a log enabled every applied gradient step (b2g_sac_step / _async, the
 *      explicit step with apply_update, b2g_sac_step_host_pipelined; replayed graphs included) appends one row of
 *      B2G_SAC_LOG_COLS floats to a device ring of `capacity` rows, at row (n_updates - 1) % capacity: policy_loss, qf1_loss,
 *      qf2_loss, value_loss, ent_coef_loss, entropy, ent_coef (after the update, as b2g_sac_metrics), learning rate.  The
 *      append is one small kernel inside the step, so the step stays free of host synchronisation.
 * metrics_log: capacity 0 disables the log (the default); a handle without a log captures and runs the step it always did.
 *   Enabling (or resizing) empties the ring and recaptures the step graphs; B2G_ESTATE while a host-pipelined step is in flight.
 * metrics_drain: waits for the handle's stream, then copies up to max_rows of the rows written since the last drain, oldest
 *   first, to rows[n][B2G_SAC_LOG_COLS]; *first_step = n_updates of the first row (row i is step *first_step + i);
 *   *lost = rows that were overwritten before this drain (skipped, never silently).  Rows past max_rows stay for the next
 *   drain.  A training-state load empties the ring.  B2G_ESTATE when the log is off.  Outputs other than rows may be NULL. */
#define B2G_SAC_LOG_COLS 8
int b2g_sac_metrics_log(b2g_sac* h, int capacity);
int b2g_sac_metrics_drain(b2g_sac* h, float* rows, int max_rows, int64_t* first_step, int* n_rows, int64_t* lost);

/* number of kernel launches one gradient step issues (bench.py's gpu_launches) */
int b2g_launches_per_step(const b2g_sac* h);
/* device-time of the last b2g_sac_step call measured with CUDA events on the handle's stream (ms) */
float b2g_last_step_ms(const b2g_sac* h);
/* per-kernel-group device time of ONE extra profiled step (events around each launch);
 * names/ms arrays of capacity cap; returns the number of groups */
int b2g_profile_step(b2g_sac* h, float lr, const char** names, float* ms, int cap);

/* ------------------------------------------------------------------------------------------------
 * BDQ (branching dueling Q-network) learner -- the `sb.BDQ` object of train_stable_baselines.py:103-104 and
 * sb_helper.py:202-226 (author's fork `bdq_sb`, absent from the reference tree: parity unpinned).
 * Variable names / shapes follow trained_models/BDQ_8pads/BDQ_simple_8pads.zip.  Actions are stored as branch
 * bin indices (floats holding integers); bin k of a branch maps to linspace(-1, 1, n_bins)[k].
 * ------------------------------------------------------------------------------------------------ */
typedef struct b2g_bdq b2g_bdq;
typedef struct b2g_bdq_cfg {
  int32_t obs_dim;             /* 100 in the shipped zips                                                */
  int32_t n_branches;          /* action dimensions (3 simplified / 5 full); <= 8                        */
  int32_t n_bins;              /* num_actions_pad (config/gripper_grasp.yaml:112)                        */
  int32_t trunk0, trunk1;      /* layers[0] = common_net                                                 */
  int32_t branch_hidden;       /* layers[1] = layers[2] (branch and state-value hidden width)            */
  int32_t batch;
  int64_t buffer_capacity;
  float gamma;
  int32_t target_update_freq;  /* hard copy every N updates (target_network_update_freq)                 */
  int32_t trunk_grad_rescale;  /* 1: scale the gradient entering the trunk by 1/(n_branches+1) (paper)   */
  uint64_t seed;
  int32_t device;
  int32_t rank, nranks;        /* data-parallel group (BASELINE config 4): each rank owns a replay shard, one NCCL
                                  all-reduce averages the gradients; nranks == 1 -> no collective                    */
  const void* nccl_id;         /* 128-byte ncclUniqueId shared by all ranks (nranks > 1)                           */
  const char* nccl_lib;        /* optional libnccl path; NULL = default search                                     */
  int32_t prioritized_replay;  /* 1: proportional prioritised replay (zip data: prioritized_replay True,
                                  config/simplified_object_picking.yaml:108-110): device sum / min segment trees   */
  float per_alpha, per_eps;    /* priority exponent (0.6) and the epsilon added to |TD| (1e-6)                     */
} b2g_bdq_cfg;
typedef struct b2g_bdq_metrics {
  float loss, mean_q, grad_norm;
  int64_t n_updates;
} b2g_bdq_metrics;

int b2g_bdq_create(const b2g_bdq_cfg* cfg, b2g_bdq** out);   /* = b2g_bdq_create2(cfg, NULL, out) */
/* replay != NULL: the transition replay keeps obs / next_obs in a pool of frame_capacity fp32 frames (frame_capacity >=
 * buffer_capacity + 1, u8_plane_mask 0, nranks 1; B2G_EINVAL otherwise), as b2g_sac_create2's replay does: every next_obs
 * takes a new frame, and row i's obs shares the frame of the previous call's next_obs of row i when the two are bitwise equal
 * (b2g_bdq_replay_add) or by construction (b2g_bdq_observe_add, unless env i was reset).  When frames run out before slots do,
 * the oldest transitions go early (b2g_bdq_replay_info counts them); sampling, uniform or prioritised, draws live slots only.
 * A training-state file records the layout: a file of the other one is refused naming replay_frames.  NULL: two fp32 rows per
 * slot, as b2g_bdq_create. */
int b2g_bdq_create2(const b2g_bdq_cfg* cfg, const b2g_replay_cfg* replay, b2g_bdq** out);
int b2g_bdq_destroy(b2g_bdq* h);
int b2g_bdq_param_count(const b2g_bdq* h);
int b2g_bdq_param_info(const b2g_bdq* h, int idx, char* name, size_t name_cap, int64_t* rows, int64_t* cols, int32_t* ndim);
int b2g_bdq_get_param(b2g_bdq* h, const char* name, float* dst, size_t numel);
int b2g_bdq_set_param(b2g_bdq* h, const char* name, const float* src, size_t numel);
int b2g_bdq_get_grad(b2g_bdq* h, const char* name, float* dst, size_t numel);
int b2g_bdq_replay_add(b2g_bdq* h, const float* obs, const float* act_idx, const float* rew, const float* next_obs,
                       const float* done, int64_t n);
int64_t b2g_bdq_replay_size(const b2g_bdq* h);
/* as b2g_replay_info: frame_capacity and live_frames are 0 without frames; bytes = b2g_transition_replay_bytes of the handle */
int b2g_bdq_replay_info(const b2g_bdq* h, int64_t* capacity, int64_t* size, int64_t* frame_capacity, int64_t* live_frames,
                        int64_t* bytes, int64_t* evicted_early);
/* the stored transition of a live slot (any output may be NULL); frame_ids[2]: the frames of its obs and next_obs (-1 without
 * frames).  B2G_EINVAL for a slot that is not live. */
int b2g_bdq_replay_get(b2g_bdq* h, int64_t slot, float* obs, float* act_idx, float* rew, float* next_obs, float* done,
                       int32_t* frame_ids);
/* On a handle that owns obs_rms (b2g_bdq_obs_rms_set, below) obs_mean / obs_var may be NULL with norm_obs != 0: the scalars
 * are set and the device statistics stay; passing them replaces the device statistics (count kept). */
int b2g_bdq_set_norm_stats(b2g_bdq* h, const double* obs_mean, const double* obs_var, double ret_var, double clip_obs,
                           double clip_rew, double eps, int norm_obs, int norm_reward);
/* n_steps x { uniform sample -> forward (online s, online s', target s') -> double-Q TD loss -> backward -> Adam ->
 * hard target copy every target_update_freq updates } */
int b2g_bdq_step(b2g_bdq* h, int n_steps, float lr, b2g_bdq_metrics* out);
/* prioritised replay: importance-sampling exponent beta of the NEXT sampled steps (SB anneals beta0 -> 1 over
 * prioritized_replay_beta_iters); last_out (may be NULL) = slots[batch], weights[batch], new priorities[batch] of the last
 * sampled step, for inspection / tests.  The slots are valid with uniform replay too (prep_kernel's Philox draw); the
 * weights and priorities are written by prioritised replay only. */
int b2g_bdq_set_per_beta(b2g_bdq* h, float beta);
int b2g_bdq_get_last_per(b2g_bdq* h, int32_t* slots, float* weights, float* priorities);
/* parity entry point: caller-supplied batch (+ optional importance weights); td_out (may be NULL): [batch, n_branches] */
int b2g_bdq_step_explicit(b2g_bdq* h, const float* obs, const float* act_idx, const float* rew, const float* next_obs,
                          const float* done, const float* weights, float lr, int apply_update, b2g_bdq_metrics* out,
                          float* td_out);
/* per-step metrics log, as b2g_sac_metrics_log / _drain: B2G_BDQ_LOG_COLS columns loss, mean_q, grad_norm (as
 * b2g_bdq_metrics), learning rate; written by b2g_bdq_step and the explicit step with apply_update */
#define B2G_BDQ_LOG_COLS 4
int b2g_bdq_metrics_log(b2g_bdq* h, int capacity);
int b2g_bdq_metrics_drain(b2g_bdq* h, float* rows, int max_rows, int64_t* first_step, int* n_rows, int64_t* lost);
/* greedy branch indices argmax_n Q_d(s, n) of the online network for n observations */
int b2g_bdq_act(b2g_bdq* h, const float* obs, int n, int32_t* act_idx_out);

/* ---- VecNormalize's observation statistics on the device and the epsilon-greedy actor fed from one upload per frame: the
 *      BDQ counterpart of b2g_sac_observe_* (same merge rule and kernel, same rule for which frames are merged, obs_rms over
 *      the flat [obs_dim] observation).  nranks == 1 only.  Up to max(batch, 256) frames per call; every call returns once the
 *      handle's stream has run what it enqueued. */
/* n raw observations (host, caller-owned), or obs == NULL to act on the observations already staged.  update_stats != 0:
 * merge them into obs_rms first (B2G_ESTATE without b2g_bdq_obs_rms_set).  act_idx_out != NULL: run the online network on
 * the staged rows normalised with the CURRENT statistics (the gather's rule: b2g_bdq_set_norm_stats's norm_obs and clip_obs),
 * take the greedy bin of every branch and, independently per (env, branch) with probability eps in [0, 1], a uniform random
 * bin instead; writes [n][n_branches] bin indices.  The random draws are Philox stream 3 under the training key at step
 * counters[7] (the number of earlier acting calls, kept in the training-state file), block env * n_branches + branch: lane x
 * explores when (x + 0.5) 2^-32 < eps (float64), lane y gives bin (y * n_bins) >> 32. */
int b2g_bdq_observe_act(b2g_bdq* h, const float* obs, int n, int update_stats, float eps, int32_t* act_idx_out);
/* Transition i = (staged obs_i, act_idx_i, rew_i, next_obs_i, done_i) into the replay (rows as b2g_bdq_replay_add stores them;
 * new rows enter the prioritised-replay trees at the running maximum priority).  next_obs is uploaded ONCE: it is this
 * transition's next observation, is merged into obs_rms when update_stats != 0 and becomes the staged observation of env i,
 * unless done_i: then reset_obs_i (the frame the auto-reset returned; the only rows of reset_obs read) is merged and staged
 * instead.  B2G_ESTATE before any b2g_bdq_observe_act; n must equal the number of staged observations. */
int b2g_bdq_observe_add(b2g_bdq* h, const float* act_idx, const float* rew, const float* next_obs, const float* done,
                        const float* reset_obs /* may be NULL when no env finished */, int n, int update_stats);
/* obs_rms in and out: float64 [obs_dim] each + count, with the checks of b2g_obs_rms_set / _get */
int b2g_bdq_obs_rms_set(b2g_bdq* h, const double* mean, const double* var, double count);
int b2g_bdq_obs_rms_get(b2g_bdq* h, double* mean, double* var, double* count);
/* bytes copied host -> device so far by b2g_bdq_observe_* and b2g_bdq_obs_rms_set (observe_bytes) and by b2g_bdq_act,
 * b2g_bdq_replay_add and b2g_bdq_set_norm_stats (other_bytes); either may be NULL */
int b2g_bdq_upload_bytes(const b2g_bdq* h, int64_t* observe_bytes, int64_t* other_bytes);
/* training state, as b2g_sac_state_save / _load: online and target parameters, Adam moments, counters, n_updates, the live
 * replay rows, the prioritised-replay sum / min trees, max priority and beta, and bdq/eps; and the device obs_rms of a handle
 * that owns one, behind one more fingerprint field (such a file loads only into a handle that owns obs_rms, and the reverse).
 * The staged observations of b2g_bdq_observe_* are not saved: a resumed run starts a fresh episode.  The fingerprint covers
 * every b2g_bdq_cfg field that decides the layout or the prioritised replay. */
int b2g_bdq_state_save(b2g_bdq* h, const char* path);
int b2g_bdq_state_load(b2g_bdq* h, const char* path);

/* ------------------------------------------------------------------------------------------------
 * Dueling double DQN learner -- the `sb.DQN` object of sb_helper.py:155-165 (stable-baselines 2.10.1 deepq, restated in
 * oracle/dqn_ref.py).  Variable names / shapes follow trained_models/DQN_4pads/DQN_simple_4pads.zip: two towers
 * deepq/model/{action_value,state_value}/fully_connected{,_1,_2} (obs -> hidden0 -> hidden1 -> n_actions / 1, ReLU),
 * Q = V + A - mean(A).  Actions are Discrete indices, stored as floats holding integers.  One step: sample (uniform or
 * prioritised) -> forward (online s, online s', target s') -> double-Q target, weighted Huber loss -> backward -> every
 * gradient tensor clipped to L2 norm 10 on its own (tf.clip_by_norm) -> TF1 Adam.  The hard target copy is
 * b2g_dqn_update_target, called by the host loop (stable-baselines counts environment steps for it, not updates).
 * ------------------------------------------------------------------------------------------------ */
typedef struct b2g_dqn b2g_dqn;
typedef struct b2g_dqn_cfg {
  int32_t obs_dim;             /* 100 in the shipped zip                                                             */
  int32_t n_actions;           /* Discrete(n): [2, 64] (12 in the shipped zip)                                       */
  int32_t hidden0, hidden1;    /* policy layers [hidden0, hidden1]: multiples of 4 in [4, 512] ([64, 64] shipped)    */
  int32_t batch;               /* <= 1024 with prioritised replay                                                    */
  int64_t buffer_capacity;
  float gamma;
  uint64_t seed;               /* Philox key of the replay draws (streams 0 and 2 of oracle/philox_ref.py)           */
  int32_t device;
  int32_t prioritized_replay;  /* 1: proportional prioritised replay on device sum / min segment trees               */
  float per_alpha, per_eps;    /* priority exponent (0.6) and the epsilon added to |td| (1e-6)                       */
} b2g_dqn_cfg;
typedef struct b2g_dqn_metrics {
  float loss;                  /* mean_b w_b huber(td_b)                                                             */
  float mean_q, mean_abs_td;   /* mean_b Q(s_b, a_b), mean_b |td_b|                                                  */
  float grad_norm;             /* global L2 norm of the gradients before the per-tensor clip                        */
  int32_t n_clipped;           /* number of gradient tensors the clip scaled                                         */
  int64_t n_updates;
} b2g_dqn_metrics;

/* B2G_EINVAL naming the limit outside n_actions in [2, 64], widths multiples of 4 in [4, 512], batch <= 65535 (<= 1024 with
 * PER) */
int b2g_dqn_create(const b2g_dqn_cfg* cfg, b2g_dqn** out);   /* = b2g_dqn_create2(cfg, NULL, out) */
/* replay: the frame pool of b2g_bdq_create2, with the same rules */
int b2g_dqn_create2(const b2g_dqn_cfg* cfg, const b2g_replay_cfg* replay, b2g_dqn** out);
int b2g_dqn_destroy(b2g_dqn* h);
/* index 0 = deepq/eps; then the online tensors, then the target tensors, in the zip's order */
int b2g_dqn_param_count(const b2g_dqn* h);
int b2g_dqn_param_info(const b2g_dqn* h, int idx, char* name, size_t name_cap, int64_t* rows, int64_t* cols, int32_t* ndim);
int b2g_dqn_get_param(b2g_dqn* h, const char* name, float* dst, size_t numel);
int b2g_dqn_set_param(b2g_dqn* h, const char* name, const float* src, size_t numel);
/* the gradient of the last step after the per-tensor clip (online tensors only) */
int b2g_dqn_get_grad(b2g_dqn* h, const char* name, float* dst, size_t numel);
/* raw transitions; every act value must be an integer in [0, n_actions) (B2G_EINVAL naming the first that is not, nothing
 * stored), as for b2g_dqn_step_explicit's batch */
int b2g_dqn_replay_add(b2g_dqn* h, const float* obs, const float* act, const float* rew, const float* next_obs, const float* done,
                       int64_t n);
int64_t b2g_dqn_replay_size(const b2g_dqn* h);
int b2g_dqn_replay_info(const b2g_dqn* h, int64_t* capacity, int64_t* size, int64_t* frame_capacity, int64_t* live_frames,
                        int64_t* bytes, int64_t* evicted_early);
int b2g_dqn_replay_get(b2g_dqn* h, int64_t slot, float* obs, float* act, float* rew, float* next_obs, float* done, int32_t* frame_ids);
/* Device bytes of the BDQ / DQN transition replay of buffer_capacity slots of obs_dim floats and act_width action floats
 * (n_branches, or 1 for DQN), without allocating it: frame_capacity * round_up(4 obs_dim, 16) + 8 buffer_capacity (frame
 * indices) with frames (frame_capacity > 0), 8 obs_dim buffer_capacity without; plus 4 (act_width + 2) buffer_capacity
 * (actions, rewards, dones).  The prioritised-replay trees are not counted. */
int64_t b2g_transition_replay_bytes(int64_t buffer_capacity, int obs_dim, int act_width, int64_t frame_capacity);
/* VecNormalize's statistics for the gather of the sampled and explicit steps (the replay holds raw transitions); not used by
 * b2g_dqn_act.  On a handle that owns obs_rms (b2g_dqn_obs_rms_set, below) obs_mean / obs_var may be NULL with norm_obs != 0:
 * the scalars are set and the device statistics stay; passing them replaces the device statistics (count kept). */
int b2g_dqn_set_norm_stats(b2g_dqn* h, const double* obs_mean, const double* obs_var, double ret_var, double clip_obs,
                           double clip_rew, double eps, int norm_obs, int norm_reward);
/* n_steps sampled steps, replayed as one captured CUDA graph each */
int b2g_dqn_step(b2g_dqn* h, int n_steps, float lr, b2g_dqn_metrics* out);
/* prioritised replay: beta of the NEXT sampled steps; slots / weights / new priorities (|td| + eps) of the last sampled step,
 * as b2g_bdq_get_last_per */
int b2g_dqn_set_per_beta(b2g_dqn* h, float beta);
int b2g_dqn_get_last_per(b2g_dqn* h, int32_t* slots, float* weights, float* priorities);
/* parity entry point: caller-supplied batch (+ optional importance weights); td_out (may be NULL): [batch] */
int b2g_dqn_step_explicit(b2g_dqn* h, const float* obs, const float* act, const float* rew, const float* next_obs, const float* done,
                          const float* weights, float lr, int apply_update, b2g_dqn_metrics* out, float* td_out);
/* per-step metrics log, as b2g_sac_metrics_log / _drain: B2G_DQN_LOG_COLS columns loss, mean_q, mean_abs_td, grad_norm,
 * n_clipped (as b2g_dqn_metrics), learning rate; written by b2g_dqn_step and the explicit step with apply_update */
#define B2G_DQN_LOG_COLS 6
int b2g_dqn_metrics_log(b2g_dqn* h, int capacity);
int b2g_dqn_metrics_drain(b2g_dqn* h, float* rows, int max_rows, int64_t* first_step, int* n_rows, int64_t* lost);
/* one device-to-device copy of the online parameters onto the target parameters */
int b2g_dqn_update_target(b2g_dqn* h);
/* greedy actions argmax_k Q(s, k) of the online network for n observations as the network sees them (a VecNormalize
 * wrapper's output: no normalisation is applied here); q_out (may be NULL): the [n, n_actions] Q rows */
int b2g_dqn_act(b2g_dqn* h, const float* obs, int n, int32_t* act_out, float* q_out);

/* ---- VecNormalize's observation statistics on the device and the epsilon-greedy actor fed from one upload per frame: the
 *      DQN counterpart of b2g_bdq_observe_* (the same observe path, merge rule and refusals, obs_rms over the flat [obs_dim]
 *      observation).  Up to max(batch, 256) frames per call; every call returns once the handle's stream has run what it
 *      enqueued.  Before any CUDA work: B2G_EINVAL for eps outside [0, 1] or an n other than the number of staged
 *      observations, B2G_ESTATE for update_stats without b2g_dqn_obs_rms_set and for b2g_dqn_observe_add before any
 *      b2g_dqn_observe_act. */
/* n raw observations (host, caller-owned), or obs == NULL to act on the observations already staged.  update_stats != 0:
 * merge them into obs_rms first.  act_out != NULL: run the online network on the staged rows normalised with the CURRENT
 * statistics (the gather's rule: b2g_dqn_set_norm_stats's norm_obs and clip_obs), take the greedy action (b2g_dqn_act's
 * argmax of Q = V + A - mean A, first maximum) and, with probability eps in [0, 1] per env, a uniform random action instead;
 * writes [n] actions.  The random draws are Philox stream 3 under the training key at step counters[7] (the number of earlier
 * acting calls, kept in the training-state file), block env: lane x explores when (x + 0.5) 2^-32 < eps (float64), lane y
 * gives action (y * n_actions) >> 32 -- b2g_bdq_observe_act's rule with one branch. */
int b2g_dqn_observe_act(b2g_dqn* h, const float* obs, int n, int update_stats, float eps, int32_t* act_out);
/* Transition i = (staged obs_i, act_i, rew_i, next_obs_i, done_i) into the replay (rows as b2g_dqn_replay_add stores them;
 * every act value must be an integer in [0, n_actions), checked before anything is stored; new rows enter the
 * prioritised-replay trees at the running maximum priority).  next_obs is uploaded ONCE: it is this transition's next
 * observation, is merged into obs_rms when update_stats != 0 and becomes the staged observation of env i, unless done_i:
 * then reset_obs_i (the frame the auto-reset returned; the only rows of reset_obs read) is merged and staged instead. */
int b2g_dqn_observe_add(b2g_dqn* h, const float* act, const float* rew, const float* next_obs, const float* done,
                        const float* reset_obs /* may be NULL when no env finished */, int n, int update_stats);
/* b2g_dqn_act on RAW observations, normalised on the device with obs_rms's table and the clip_obs / norm_obs of
 * b2g_dqn_set_norm_stats: predict while the learner owns the statistics.  B2G_ESTATE without b2g_dqn_obs_rms_set. */
int b2g_dqn_act_raw(b2g_dqn* h, const float* obs, int n, int32_t* act_out, float* q_out);
/* obs_rms in and out: float64 [obs_dim] each + count, with the checks of b2g_obs_rms_set / _get */
int b2g_dqn_obs_rms_set(b2g_dqn* h, const double* mean, const double* var, double count);
int b2g_dqn_obs_rms_get(b2g_dqn* h, double* mean, double* var, double* count);
/* bytes copied host -> device so far by b2g_dqn_observe_* and b2g_dqn_obs_rms_set (observe_bytes) and by b2g_dqn_act /
 * _act_raw, b2g_dqn_replay_add and b2g_dqn_set_norm_stats (other_bytes); either may be NULL */
int b2g_dqn_upload_bytes(const b2g_dqn* h, int64_t* observe_bytes, int64_t* other_bytes);
/* training state, as b2g_bdq_state_save / _load: parameters, Adam moments, counters, n_updates, the live replay rows, the
 * prioritised-replay trees, max priority and beta, and deepq/eps; and the device obs_rms of a handle that owns one, behind
 * one more fingerprint field (such a file loads only into a handle that owns obs_rms, and the reverse; a handle without
 * device statistics writes the files it wrote before).  The staged observations of b2g_dqn_observe_* are not saved.  The
 * fingerprint covers every b2g_dqn_cfg field that decides the layout or the prioritised replay. */
int b2g_dqn_state_save(b2g_dqn* h, const char* path);
int b2g_dqn_state_load(b2g_dqn* h, const char* path);

/* ------------------------------------------------------------------------------------------------
 * PPO2 learner -- the `sb.PPO2` object of sb_helper.py:137-154 (stable-baselines 2.10.1 ppo2 with common.policies.MlpPolicy,
 * restated in oracle/ppo_ref.py).  Variables model/{pi_fc0,vf_fc0,pi_fc1,vf_fc1,vf,pi}/{w,b}, model/pi/logstd [1, A] and the
 * untrained head model/q/{w,b}: two tanh towers obs -> hidden0 -> hidden1, a diagonal Gaussian (mean pi, state-independent
 * logstd) and the value vf.  The rollout lives on the device: b2g_ppo_rollout_act / _reward fill n_steps rows of n_envs
 * environments, b2g_ppo_update runs GAE and noptepochs x nminibatches clipped-surrogate minibatch steps (global-norm gradient
 * clip, TF1 Adam with epsilon 1e-5) in the caller's permutation, as one CUDA graph.
 * ------------------------------------------------------------------------------------------------ */
typedef struct b2g_ppo b2g_ppo;
typedef struct b2g_ppo_cfg {
  int32_t obs_dim;             /* flattened observation (float32, no scaling): [1, 65536]                            */
  int32_t n_actions;           /* Box action size: [1, 16]                                                            */
  int32_t hidden0, hidden1;    /* net_arch pi = vf = [hidden0, hidden1]: multiples of 4 in [4, 256] ([64, 64] default)  */
  int32_t n_envs;              /* [1, 4096]                                                                           */
  int32_t n_steps;             /* rollout length per env (128 default)                                                */
  int32_t nminibatches;        /* divides n_batch = n_steps * n_envs; minibatch n_batch / nminibatches <= 16384       */
  int32_t noptepochs;          /* noptepochs * nminibatches <= 4096                                                   */
  float gamma, lam;            /* discount and GAE lambda (0.99, 0.95)                                                */
  float ent_coef, vf_coef;     /* 0.01, 0.5                                                                           */
  float max_grad_norm;         /* tf.clip_by_global_norm bound (0.5)                                                  */
  uint64_t seed;               /* the actor's noise key is seed ^ 0xA5A5A5A5DEADBEEF (Philox stream 1)               */
  int32_t device;
} b2g_ppo_cfg;
typedef struct b2g_ppo_metrics {
  float policy_loss, value_loss, entropy, approxkl, clipfrac;   /* ppo2.py's logged losses (update: mean over minibatches) */
  float grad_norm;             /* global L2 norm of the gradient before the clip                                      */
  int64_t n_updates;           /* minibatch steps applied so far                                                      */
} b2g_ppo_metrics;

/* B2G_EINVAL naming the limit outside the ranges above */
int b2g_ppo_create(const b2g_ppo_cfg* cfg, b2g_ppo** out);
int b2g_ppo_destroy(b2g_ppo* h);
/* the 15 variables in the zip's order (model/ prefix); q/w and q/b are never updated */
int b2g_ppo_param_count(const b2g_ppo* h);
int b2g_ppo_param_info(const b2g_ppo* h, int idx, char* name, size_t name_cap, int64_t* rows, int64_t* cols, int32_t* ndim);
int b2g_ppo_get_param(b2g_ppo* h, const char* name, float* dst, size_t numel);
int b2g_ppo_set_param(b2g_ppo* h, const char* name, const float* src, size_t numel);
/* the gradient of the last minibatch step after the global-norm clip (trained variables only) */
int b2g_ppo_get_grad(b2g_ppo* h, const char* name, float* dst, size_t numel);
/* rollout step t: obs [n_envs, obs_dim] -> row t; act_out [n_envs, n_actions] = mean + exp(logstd) * eps, unclipped (the
 * caller clips for the env); action, value and neglogp stay in row t.  B2G_ESTATE when n_steps rows are filled. */
int b2g_ppo_rollout_act(b2g_ppo* h, const float* obs, float* act_out);
/* rewards [n_envs] of step t and the episode-start flags of step t + 1 (the env's done flags) */
int b2g_ppo_rollout_reward(b2g_ppo* h, const float* rew, const float* done);
/* empty rollout, episode-start flags cleared (a fresh episode) */
int b2g_ppo_rollout_reset(b2g_ppo* h);
/* [n_steps, n_envs] (time-major) advantages and returns of the last update's GAE, values, neglogp, actions [.., n_actions];
 * any pointer may be NULL */
int b2g_ppo_rollout_get(b2g_ppo* h, float* adv, float* ret, float* val, float* nlp, float* act);
/* one update on a full rollout: last_obs [n_envs, obs_dim] bootstraps the GAE; perm [noptepochs * n_batch] holds each epoch's
 * permutation of the env-major flattened batch; cliprange_vf < 0 turns value clipping off.  out: means over the minibatches. */
int b2g_ppo_update(b2g_ppo* h, const float* last_obs, const int32_t* perm, float lr, float cliprange, float cliprange_vf,
                   b2g_ppo_metrics* out);
/* parity entry point: one minibatch [n_batch / nminibatches] supplied by the caller (advantages = returns - values) */
int b2g_ppo_train_step_explicit(b2g_ppo* h, const float* obs, const float* returns, const float* actions, const float* values,
                                const float* neglogp, float lr, float cliprange, float cliprange_vf, int apply_update,
                                b2g_ppo_metrics* out);
/* predict: n observations -> mean (deterministic) or mean + std * eps (stream 1, advancing the same counter as the rollout);
 * nothing is written to the rollout.  value_out / neglogp_out may be NULL. */
int b2g_ppo_act(b2g_ppo* h, const float* obs, int n, int deterministic, float* act_out, float* value_out, float* neglogp_out);
/* Adam step, stream-1 step counter, rollout rows filled */
int b2g_ppo_get_step(b2g_ppo* h, int64_t* adam_step, int64_t* noise_step, int32_t* rollout_rows);
/* training state at an update boundary: parameters (q included), Adam moments, counters, n_updates.  A load empties the
 * rollout and clears the episode-start flags. */
int b2g_ppo_state_save(b2g_ppo* h, const char* path);
int b2g_ppo_state_load(b2g_ppo* h, const char* path);

/* ---- VecNormalize's observation statistics on the device and the rollout fed from one upload per frame (PPO2 and TRPO
 *      share these bodies; nranks is 1).  obs_rms is float64 [obs_dim] mean / var + count with the merge rule, kernel and
 *      checks of b2g_obs_rms_set / _get.  Each observation is normalised ONCE, right after its merge, and stored in the rollout
 *      as VecNormalize returns it: float(clip((double(x) - mean) / sqrt(var + epsilon), -clip_obs, clip_obs)), evaluated in
 *      float64 in numpy's order and rounded once (bit-identical to VecNormalize.normalize_obs on the same statistics); without
 *      obs_rms, or with norm_obs 0, the rows are stored as given.  The statistics also ride the training-state file (an ORMS
 *      section behind the obs_rms fingerprint field; a file of the other kind is refused naming obs_rms). */
int b2g_ppo_obs_rms_set(b2g_ppo* h, const double* mean, const double* var, double count);
int b2g_ppo_obs_rms_get(b2g_ppo* h, double* mean, double* var, double* count);
/* bytes copied host -> device by b2g_ppo_observe_act and b2g_ppo_obs_rms_set (observe_bytes) and by b2g_ppo_act_raw (other) */
int b2g_ppo_upload_bytes(const b2g_ppo* h, int64_t* observe_bytes, int64_t* other_bytes);
/* VecNormalize's clip_obs, epsilon and norm_obs for the normalisation (defaults 10, 1e-8, 1); B2G_EINVAL unless clip_obs and
 * epsilon are finite and >= 0 */
int b2g_ppo_set_norm_stats(b2g_ppo* h, double clip_obs, double eps, int norm_obs);
/* obs != NULL: n = n_envs raw frames (host, caller-owned) are uploaded once, merged into obs_rms when update_stats != 0
 * (B2G_ESTATE without b2g_ppo_obs_rms_set) and normalised into the current rollout row: row t, or row t + 1 once row t's action
 * is drawn (so the frames the env returns after step t go to row t + 1, and after the last step to row n_steps, the bootstrap
 * row).  act_out != NULL: rollout step t on that row (b2g_ppo_rollout_act without the upload; B2G_ESTATE when row t holds no
 * staged observation or its action is drawn).  Both NULL: B2G_EINVAL.  n != n_envs: B2G_EINVAL.  One stream synchronise.
 * b2g_ppo_update with last_obs == NULL bootstraps from the staged row n_steps and starts the next rollout from it (row 0);
 * without one it is refused with B2G_EINVAL. */
int b2g_ppo_observe_act(b2g_ppo* h, const float* obs, int n, int update_stats, float* act_out);
/* b2g_ppo_act on raw observations: normalised with the current statistics first (nothing is merged) */
int b2g_ppo_act_raw(b2g_ppo* h, const float* obs, int n, int deterministic, float* act_out, float* value_out, float* neglogp_out);

/* ------------------------------------------------------------------------------------------------
 * TRPO learner -- the `sb.TRPO` object of sb_helper.py:129-136 (stable-baselines 2.10.1 trpo_mpi with common.policies.MlpPolicy
 * and one environment, restated in tests/trpo_ref.py).  Variables pi/model/... (the live policy, PPO2's 15 variables under
 * pi/) then oldpi/model/... (the old policy, the same 15).  The rollout of timesteps_per_batch = N steps lives on the device
 * (b2g_trpo_rollout_act / _reward); b2g_trpo_update runs, as one CUDA graph: the boundary action and bootstrap value, GAE,
 * oldpi := pi, the policy gradient at theta_old, cg_iters conjugate-gradient iterations on Fisher-vector products over the
 * rows [::5], the KL-constrained line search (ten step sizes 0.5^k in one pass), then vf_iters passes of 128-row value
 * minibatches with MpiAdam (epsilon 1e-8).  Box actions only.
 * ------------------------------------------------------------------------------------------------ */
typedef struct b2g_trpo b2g_trpo;
typedef struct b2g_trpo_cfg {
  int32_t obs_dim;             /* flattened observation (float32, no scaling): [1, 65536]                            */
  int32_t n_actions;           /* Box action size: [1, 16]                                                            */
  int32_t hidden0, hidden1;    /* net_arch pi = vf = [hidden0, hidden1]: multiples of 4 in [4, 256] ([64, 64] default)  */
  int32_t timesteps_per_batch; /* N: [1, 16384] (1024 default)                                                       */
  int32_t cg_iters;            /* [1, 64] (10)                                                                        */
  int32_t vf_iters;            /* [0, 64] (3)                                                                         */
  float gamma, lam;            /* 0.99, 0.98                                                                          */
  float max_kl;                /* > 0 (0.01)                                                                          */
  float cg_damping;            /* >= 0 (1e-2)                                                                         */
  float entcoeff;              /* 0                                                                                   */
  float vf_stepsize;           /* MpiAdam learning rate (3e-4)                                                        */
  uint64_t seed;               /* the actor's noise key is seed ^ 0xA5A5A5A5DEADBEEF (Philox stream 1)               */
  int32_t device;
} b2g_trpo_cfg;
typedef struct b2g_trpo_metrics {
  float optimgain, meankl, entbonus, surrgain, entropy;   /* the losses at theta_old                                   */
  float optimgain_after, meankl_after, entbonus_after, surrgain_after, entropy_after;  /* at the accepted theta          */
  float grad_sq;               /* g . g of the policy gradient at theta_old                                          */
  float shs;                   /* 0.5 stepdir . F stepdir                                                            */
  float expected_improve;      /* g . fullstep                                                                       */
  float vf_loss;               /* mean value loss over the value minibatches (0 without any)                         */
  int32_t cg_iters;            /* conjugate-gradient iterations run                                                  */
  int32_t accepted;            /* line-search k (step 0.5^k), -1: every candidate rejected, -2: zero gradient       */
  int64_t n_iterations;        /* policy iterations so far                                                           */
} b2g_trpo_metrics;

/* B2G_EINVAL naming the limit outside the ranges above, or the device memory the line search needs */
int b2g_trpo_create(const b2g_trpo_cfg* cfg, b2g_trpo** out);
int b2g_trpo_destroy(b2g_trpo* h);
/* the 30 variables in the zip's order: pi/model/... then oldpi/model/...; get_grad returns the policy gradient g at theta_old
 * of the last step for the policy variables (pi_fc0, pi_fc1, pi and pi/logstd under pi/model/) and refuses the others */
int b2g_trpo_param_count(const b2g_trpo* h);
int b2g_trpo_param_info(const b2g_trpo* h, int idx, char* name, size_t name_cap, int64_t* rows, int64_t* cols, int32_t* ndim);
int b2g_trpo_get_param(b2g_trpo* h, const char* name, float* dst, size_t numel);
int b2g_trpo_set_param(b2g_trpo* h, const char* name, const float* src, size_t numel);
int b2g_trpo_get_grad(b2g_trpo* h, const char* name, float* dst, size_t numel);
/* rollout step t: obs [obs_dim] -> row t; act_out [n_actions] = mean + exp(logstd) * eps, unclipped.  After an update, step 0
 * returns the action drawn for the boundary observation before that update (stable-baselines' traj_segment_generator) and
 * draws nothing.  B2G_ESTATE when N rows are filled. */
int b2g_trpo_rollout_act(b2g_trpo* h, const float* obs, float* act_out);
/* the reward of step t and the env's done flag after it */
int b2g_trpo_rollout_reward(b2g_trpo* h, float rew, float done);
/* empty rollout, episode-start flag cleared, no carried action (a fresh env.reset()) */
int b2g_trpo_rollout_reset(b2g_trpo* h);
/* [N] advantages, tdlamret, values and [N, n_actions] actions of the rollout; any pointer may be NULL */
int b2g_trpo_rollout_get(b2g_trpo* h, float* adv, float* ret, float* val, float* act);
/* one iteration on a full rollout: last_obs [obs_dim] is the boundary observation; perm [vf_iters * N] holds each value pass's
 * permutation.  B2G_ESTATE when the conjugate-gradient step direction is not finite (metrics are still written). */
int b2g_trpo_update(b2g_trpo* h, const float* last_obs, const int32_t* perm, b2g_trpo_metrics* out);
/* test entry points, at the current parameters; both empty the rollout.  fvp: v [n_policy] in var_list order (pi_fc0/w,
 * pi_fc0/b, pi_fc1/w, pi_fc1/b, pi/w, pi/b, pi/logstd) -> F v over the rows [::5] of obs [N, obs_dim], damping included.
 * step_explicit: the policy and value step of b2g_trpo_update on obs [N, obs_dim], actions [N, n_actions], raw advantages
 * [N], tdlamret [N] and perm [vf_iters * N]; grad / stepdir / fullstep [n_policy] in var_list order may be NULL. */
int b2g_trpo_fvp(b2g_trpo* h, const float* obs, const float* v, float* out);
int b2g_trpo_step_explicit(b2g_trpo* h, const float* obs, const float* actions, const float* adv, const float* tdlamret,
                           const int32_t* perm, b2g_trpo_metrics* out, float* grad, float* stepdir, float* fullstep);
/* predict: n observations -> mean (deterministic) or mean + std * eps (stream 1, advancing the rollout's counter);
 * value_out may be NULL */
int b2g_trpo_act(b2g_trpo* h, const float* obs, int n, int deterministic, float* act_out, float* value_out);
/* value-Adam step, stream-1 step counter, rollout rows filled */
int b2g_trpo_get_step(b2g_trpo* h, int64_t* adam_step, int64_t* noise_step, int32_t* rollout_rows);
/* training state at an iteration boundary: parameters (pi and oldpi), the value Adam's moments, counters, iterations.  A load
 * empties the rollout and clears the episode-start flag. */
int b2g_trpo_state_save(b2g_trpo* h, const char* path);
int b2g_trpo_state_load(b2g_trpo* h, const char* path);
/* the PPO2 observe path above on the TRPO handle (n = 1).  After an update, step 0 acts on the carried boundary row: the
 * normalised row as it was staged, and the action drawn for it before the update. */
int b2g_trpo_obs_rms_set(b2g_trpo* h, const double* mean, const double* var, double count);
int b2g_trpo_obs_rms_get(b2g_trpo* h, double* mean, double* var, double* count);
int b2g_trpo_upload_bytes(const b2g_trpo* h, int64_t* observe_bytes, int64_t* other_bytes);
int b2g_trpo_set_norm_stats(b2g_trpo* h, double clip_obs, double eps, int norm_obs);
int b2g_trpo_observe_act(b2g_trpo* h, const float* obs, int n, int update_stats, float* act_out);
int b2g_trpo_act_raw(b2g_trpo* h, const float* obs, int n, int deterministic, float* act_out, float* value_out);

/* ------------------------------------------------------------------------------------------------------------
 * Row a12: auto-encoder ENCODER forward (perception for the `encoded depth` observation, SURVEY.md section 8).
 * Replaces SimpleAutoEncoder.encode  (/root/reference/manipulation_main/gripperEnv/encoders.py:59-61; graph :87-108)
 * called per env step from EncodedDepthImgSensor.get_state (manipulation_main/gripperEnv/sensor.py:218-222).
 * Layer spec = config.yaml `network` (filters / kernel_size / strides, padding 'same'), LeakyReLU(alpha) after every
 * conv and after Dense(encoding_dim).  Weights are the Keras arrays from model.h5: conv kernels [k,k,in,out], dense
 * kernel [flat,out] (flatten order H,W,C), biases [out].  Any alpha is accepted (the forward applies it as given).
 * b2g_encoder_create returns B2G_EINVAL, before it touches a device, for a bad layer spec, hidden filter counts that are
 * not multiples of 4, a flattened size that is not a multiple of 4, or a max_batch at which any layer's zero-bordered
 * input (the dense layer's input included) holds more than 2^31 - 1 floats.
 * ------------------------------------------------------------------------------------------------------------ */
#define B2G_ENC_MAX_LAYERS 8
typedef struct b2g_encoder b2g_encoder;
typedef struct b2g_encoder_cfg {
  int32_t height, width, channels;      /* Input(shape=(64, 64, 1)) in the reference */
  int32_t n_layers;                     /* conv layers */
  int32_t filters[B2G_ENC_MAX_LAYERS];
  int32_t kernel[B2G_ENC_MAX_LAYERS];
  int32_t strides[B2G_ENC_MAX_LAYERS];
  int32_t encoding_dim;
  float alpha;                          /* LeakyReLU slope, config.get('alpha', 0.1) */
  int32_t max_batch;
  int32_t device;
} b2g_encoder_cfg;
int b2g_encoder_create(const b2g_encoder_cfg* cfg, b2g_encoder** out);      /* = create2(cfg, B2G_PREC_FP32_SIMT, out) */
/* The encoder at a chosen precision (b2g_encoder_encode, and the stage b2g_*_set_obs_encoder copies from it, run at it):
 *   B2G_PREC_FP32_SIMT  fp32 FFMA gather-GEMMs on the CUDA cores (the default; what b2g_encoder_create builds);
 *   B2G_PREC_BF16X3     the four contractions on the wgmma engine: operands split into BF16 hi + lo, hi*hi + hi*lo + lo*hi
 *                       summed in fp32 (about 2^-16 relative per layer, the SAC learner's bf16x3 contract).  Layer 0 reads an
 *                       x-unfolded copy of the image whose kernel rows are padded to a multiple of 8 taps; every conv but the
 *                       last needs filters % 8 == 0.  A frame's encoding does not depend on its batch or its row in it.
 * B2G_EINVAL before any CUDA call for B2G_PREC_BF16 (single-pass BF16 encodings are not offered as policy inputs), any other
 * value, a geometry b2g_encoder_create refuses, and a bf16x3 geometry the engine cannot take (the message names the reason). */
int b2g_encoder_create2(const b2g_encoder_cfg* cfg, int32_t precision, b2g_encoder** out);
int b2g_encoder_destroy(b2g_encoder* h);
int b2g_encoder_n_layers(const b2g_encoder* h);                      /* conv layers + 1 (dense) */
int b2g_encoder_layer_shape(const b2g_encoder* h, int layer, int64_t* kernel_numel, int64_t* bias_numel);
int b2g_encoder_set_weights(b2g_encoder* h, int layer, const float* kernel, size_t kernel_numel, const float* bias,
                            size_t bias_numel);
/* imgs: host [n, height, width, channels] fp32 -> out: host [n, encoding_dim]; B2G_ESTATE until every layer is loaded */
int b2g_encoder_encode(b2g_encoder* h, const float* imgs, int n, float* out);
/* debug: b2g_encoder_encode of imgs, then every layer's output as the next layer reads it (bf16x3: hi + lo of its planes):
 * out = [conv 0 [n][out_h][out_w][f] | conv 1 ... | dense [n][encoding_dim]], out_numel their total */
int b2g_debug_encoder_layers(b2g_encoder* h, const float* imgs, int n, float* out, int64_t out_numel);

/* ---- the encoder on a learner's observe path: the env hands out raw depth rows and the learner encodes them on its device.
 * enc != NULL attaches: the encoder's geometry and weights are copied device to device into a stage the learner handle owns,
 * on the handle's device and stream, for up to max(batch, 256) rows (the observe calls' limit); the weights are frozen and
 * the encoder handle may be destroyed afterwards.  enc == NULL detaches.  Either way the staged observations are cleared.
 * With an encoder attached, b2g_sac_observe_act / _add (and the BDQ pair) take RAW rows [n][H*W*C + tail]: pixels in HWC
 * order, then `tail` floats (the actuator state, a time feature) copied to columns [encoding_dim, obs_dim) of the encoded
 * row.  Only the n frames and the reset frames of finished envs cross the bus, and only those are encoded; obs_rms, the actor
 * and the replay then work on encoded rows [obs_dim] exactly as before, so b2g_sac_act, b2g_replay_add, the step and the
 * training-state file are unchanged.  The upload counters count the raw bytes.
 * Before any CUDA call: B2G_EINVAL for a CNN SAC policy, encoding_dim + tail != obs_dim, tail < 0 or an encoder on another
 * device; B2G_ESTATE for an encoder layer without weights or nranks > 1. */
int b2g_sac_set_obs_encoder(b2g_sac* h, const b2g_encoder* enc, int tail);
int b2g_bdq_set_obs_encoder(b2g_bdq* h, const b2g_encoder* enc, int tail);
/* the same on the DQN handle: b2g_dqn_observe_act / _add take raw rows */
int b2g_dqn_set_obs_encoder(b2g_dqn* h, const b2g_encoder* enc, int tail);
/* the same on the PPO2 and TRPO handles: b2g_ppo_observe_act / b2g_trpo_observe_act take raw rows, encode them into the
 * staged rows and normalise those into the rollout */
int b2g_ppo_set_obs_encoder(b2g_ppo* h, const b2g_encoder* enc, int tail);
int b2g_trpo_set_obs_encoder(b2g_trpo* h, const b2g_encoder* enc, int tail);

/* ------------------------------------------------------------------------------------------------------------
 * Auto-encoder TRAINING (encoders.py:40-61 train / test / predict, graph :84-136): the full Keras model
 * encoder -> decoder on one handle, trained with mean_squared_error and Keras Adam (eps 1e-7) in fp32 on the GPU.
 * Decoder: Dense(h*w*c) + LeakyReLU, Reshape, then for i = L-1..1 UpSampling2D(strides_i) + Conv2D(filters_{i-1},
 * kernel_i, 'same') + LeakyReLU, then UpSampling2D(strides_0) + Conv2D(1, kernel_0, 'same').
 * Layers are numbered in model.h5 order: encoder convs, encoder dense, decoder dense, decoder convs, output conv
 * (2 * n_layers + 2); weights use the Keras layouts of b2g_encoder_set_weights.  Requires channels == 1, every filter
 * count a multiple of 4 and a decoder that returns to height x width (else B2G_EINVAL).  alpha must be finite and >= 0:
 * the backward reads the LeakyReLU derivative from the sign of the stored output, which cannot tell a negative
 * pre-activation from a positive one when alpha < 0.  The output conv (1 filter, kernel_0, filters_0 inputs) needs
 * kernel_0^2 * filters_0 <= 2048 and (kernel_0^2 * filters_0 + (kernel_0 + 7)^2 * (filters_0 + 1)) * 4 <= 98304 bytes of
 * shared memory.  Every one of these refusals comes before any device is touched.  max_batch is the largest
 * batch of any call.  Calls that run the model return B2G_ESTATE until every layer has weights.
 * ------------------------------------------------------------------------------------------------------------ */
typedef struct b2g_autoencoder b2g_autoencoder;
int b2g_autoencoder_create(const b2g_encoder_cfg* cfg, b2g_autoencoder** out);     /* = create2(cfg, B2G_PREC_FP32_SIMT, out) */
/* The training handle at a chosen precision (b2g_autoencoder_step, _train_epoch, _evaluate and _predict all run at it):
 *   B2G_PREC_FP32_SIMT  every contraction's exact fp32 products summed in double on the CUDA cores (what _create builds);
 *   B2G_PREC_BF16X3     every conv and dense contraction whose operands come in 16-byte groups of 4 values on the wgmma
 *                       engine: operands split into BF16 hi + lo in registers, hi*hi + hi*lo + lo*hi summed in fp32 per
 *                       64-row chunk; weight-gradient split-R partials (and the bias gradients' fp32 partial column sums)
 *                       added into the double gradient arena with double atomics.  conv1's forward and weight gradient (one
 *                       input channel) and the output conv (one filter) stay on the CUDA cores.  Each element is within
 *                       about 2^-15 of the sum of |products| of its contraction, not of its value: conv1's kernel gradient,
 *                       a sum whose terms cancel by a factor of several hundred, is correspondingly less precise.
 * B2G_EINVAL before any CUDA call for B2G_PREC_BF16 (single-pass BF16 training is not offered), any other value and every
 * geometry _create refuses; bf16x3 accepts every geometry _create accepts (filters % 4 == 0 gives the 4-value groups). */
int b2g_autoencoder_create2(const b2g_encoder_cfg* cfg, int32_t precision, b2g_autoencoder** out);
int b2g_autoencoder_destroy(b2g_autoencoder* h);
int b2g_autoencoder_n_layers(const b2g_autoencoder* h);
int b2g_autoencoder_layer_shape(const b2g_autoencoder* h, int layer, int64_t* kernel_numel, int64_t* bias_numel);
int b2g_autoencoder_set_weights(b2g_autoencoder* h, int layer, const float* kernel, size_t kernel_numel, const float* bias,
                                size_t bias_numel);
int b2g_autoencoder_get_weights(b2g_autoencoder* h, int layer, float* kernel, size_t kernel_numel, float* bias, size_t bias_numel);
/* gradients of the last b2g_autoencoder_step (mean squared error over the batch) */
int b2g_autoencoder_get_grad(b2g_autoencoder* h, int layer, float* kernel, size_t kernel_numel, float* bias, size_t bias_numel);
/* zeroes Adam's moments and its step count */
int b2g_autoencoder_reset_optimizer(b2g_autoencoder* h);
/* copies n images [n, height, width, 1] to the device; targets == NULL trains towards the inputs themselves */
int b2g_autoencoder_set_dataset(b2g_autoencoder* h, const float* inputs, const float* targets, int64_t n);
/* one pass over dataset rows order[0..n_order) in batches of `batch` (the last one may be partial): one Adam step per batch;
 * *mean_loss = sample-weighted mean of the batch losses, each taken before its update */
int b2g_autoencoder_train_epoch(b2g_autoencoder* h, const int32_t* order, int64_t n_order, int batch, float lr, double* mean_loss);
/* mean squared error over dataset rows [start, start + count) */
int b2g_autoencoder_evaluate(b2g_autoencoder* h, int64_t start, int64_t count, double* mean_loss);
/* imgs: host [n, height, width, 1] -> out: host [n, height, width, 1] reconstructions */
int b2g_autoencoder_predict(b2g_autoencoder* h, const float* imgs, int n, float* out);
/* one step on a host batch (targets == NULL: the inputs); apply_update == 0 only computes loss and gradients */
int b2g_autoencoder_step(b2g_autoencoder* h, const float* inputs, const float* targets, int n, float lr, int apply_update,
                         double* loss);
/* debug: a device tensor of layer `layer` as the last call left it, the whole max_batch buffer copied to out (numel elements):
 * which = 0 the input the layer's contractions read (convs: the zero-bordered NHWC buffer [N][hp][wp][in_c], a decoder conv's
 * holding the upsampled map; dense: rows [N][in_ld]), 1 the stored LeakyReLU output where no bordered buffer holds it
 * (encoder dense [N][round4(encoding_dim)], decoder dense [N][h*w*c], decoder convs [N][out_h][out_w][f]), 2 the gradient of
 * the pre-activation (convs: [N][in_h + pad_t + k - 1][in_w + pad_l + k - 1][f] with output (oy, ox) at (oy*s + k-1,
 * ox*s + k-1); dense: rows [N][round4(f)]).  on_tc (optional, 3 ints) receives whether the layer's forward, input gradient and
 * weight gradient run on the wgmma engine (1), on the CUDA cores (0) or not as a contraction (-1).  out == NULL only fills
 * on_tc.  b2g_debug_autoencoder_tensor_numel gives numel (-1: no such tensor). */
int b2g_debug_autoencoder_tensor(b2g_autoencoder* h, int layer, int which, float* out, int64_t numel, int32_t* on_tc);
int64_t b2g_debug_autoencoder_tensor_numel(b2g_autoencoder* h, int layer, int which);

/* ------------------------------------------------------------------------------------------------------------
 * Bring-up hook (not on the product path): C[M,N] = A[M,K] * B[N,K]^T through the wgmma engine; host pointers,
 * K a multiple of 8; x3 != 0 -> BF16 hi/lo split (3 MMAs); split_k > 1 -> that many partial accumulators summed
 * with fp32 atomics.  tools/tc_accum_probe.py uses it to measure the accumulation behaviour of the tensor core.
 * ------------------------------------------------------------------------------------------------------------ */
int b2g_debug_gemm(int M, int N, int K, const float* A, const float* B, float* C, int x3, int split_k);

/* Bring-up hook (not on the product path): one grouped launch of the fp32 gather-GEMM engine (csrc/gg_simt.cu) over problems
 * the caller describes, through build 0 (plain fp32), 1 (sums in double, GG_EPI_LRELU_GRAD and m-direction GG_A_SCALAR; the
 * auto-encoder's build) or 2 (GG_EPI_BIAS_TANH / GG_EPI_TANH_GRAD; PPO2's build).  Problem p computes
 *   C[cM[m] + cN[n]]  (=|+=)  epi( sum_r  A[aM[m] + aR[r]] * B[bR[r] + bN[n]] )
 * with every operand an element offset into one of four host arenas: A, B, C, bias, mask and colsum into f32 (C and colsum
 * into f64 under build 1 with GG_EPI_ATOMIC / GG_COLSUM), the tables aM .. kN into tabs (kM / kN = -1: the engine's default
 * cM / cN), C_hi / C_lo into u16 (-1: none; both or neither).  The f32, f64 and u16 arenas are uploaded, the tiles laid out
 * as the handles lay them out, the group launched once on a stream of its own, and the three arenas copied back.
 * Before any CUDA call, B2G_EINVAL (b2g_last_error names the broken contract) refuses: n outside 1..16; M, N, R < 1,
 * splitR < 1 or > R, splitR > 1 without GG_EPI_ATOMIC; a flag the build does not have; a missing operand; an address any
 * table can reach outside its arena; GG_A_RVEC / GG_B_RVEC without r contiguous in aligned 4-groups (16-byte addresses),
 * except A under GG_A_SCALAR; an m- (n-) direction operand whose full aligned 4-groups of rows (columns) are not contiguous
 * and 16-byte aligned, except A under build 1 with GG_A_SCALAR; GG_COLSUM with GG_B_RVEC (the column sums are taken from the
 * n-direction B loads); C_hi / C_lo with GG_EPI_ATOMIC; C not 16-byte aligned.  Arena lengths are element counts below 2^31.  Flag values: */
#define B2G_GG_A_RVEC (1 << 0)
#define B2G_GG_B_RVEC (1 << 1)
#define B2G_GG_EPI_BIAS_RELU (1 << 2)
#define B2G_GG_EPI_MASK (1 << 3)
#define B2G_GG_EPI_ATOMIC (1 << 4)
#define B2G_GG_COLSUM (1 << 5)
#define B2G_GG_EPI_BIAS (1 << 10)
#define B2G_GG_EPI_SCALE (1 << 11)
#define B2G_GG_A_SCALAR (1 << 12)
#define B2G_GG_EPI_BIAS_LRELU (1 << 13)
#define B2G_GG_EPI_LRELU_GRAD (1 << 15)
#define B2G_GG_EPI_BIAS_TANH (1 << 16)
#define B2G_GG_EPI_TANH_GRAD (1 << 17)
typedef struct {
  int64_t A, B, C, bias, mask, colsum;       /* offsets into f32 (C / colsum: f64 under build 1 with ATOMIC / COLSUM); -1 = none */
  int64_t aM, aR, bR, bN, cM, cN, kM, kN;    /* offsets into tabs; kM / kN -1 = cM / cN */
  int64_t C_hi, C_lo;                        /* offsets into u16, -1 = none */
  int32_t M, N, R, flags, splitR;
  float alpha;                               /* GG_EPI_SCALE factor, LeakyReLU slope */
} b2g_debug_gg_problem;
int b2g_debug_gg_simt(int build, const b2g_debug_gg_problem* p, int n, float* f32, int64_t n_f32, double* f64, int64_t n_f64,
                      uint16_t* u16, int64_t n_u16, const int32_t* tabs, int64_t n_tabs);

/* Bring-up hook (not on the product path): one grouped launch of the wgmma gather-GEMM engine (csrc/gg_tc.cu) over 1 to 16
 * problems the caller describes; x3 = 1 multiplies hi*hi + hi*lo + lo*hi of the BF16 operand splits, x3 = 0 hi*hi only.
 * Problem p computes C[cM[m] + cN[n]] (=|+=) epi( sum_r A[aM[m] + aR[r]] * B[bR[r] + bN[n]] ) from fp32 A and B (offsets into
 * f32), or under B2G_GG_PLANES from BF16 planes A_hi / A_lo / B_hi / B_lo (offsets into u16; the plane B of a K-major problem
 * reads through bR_p / bN_p when given).  C, bias, mask and colsum are offsets into f32, C_hi / C_lo into u16 (-1: none), the
 * tables into tabs (kM / kN -1: cM / cN).  GG_CN_AFFINE4 and the column-table ids are derived from the tables as the SAC
 * handle derives them; the tiles are laid out as the handle lays them out (splitR is the caller's).  The arenas are uploaded,
 * the group launched once on a stream of its own, and f32 and u16 copied back.
 * Before any CUDA call, B2G_EINVAL (b2g_last_error names the broken contract) refuses: x3 not 0 or 1; n outside 1..16;
 * problems whose flags select different kernels (B2G_GG_PLANES, else B2G_GG_A_RVEC | B2G_GG_B_RVEC); a flag the engine does not
 * implement (only A_RVEC, B_RVEC, EPI_BIAS_RELU, EPI_MASK, EPI_ATOMIC, COLSUM, PLANES, A_ALIGN4, MN_MAJOR and A_ROWLANES are);
 * A_ALIGN4, MN_MAJOR or A_ROWLANES without PLANES; COLSUM with B_RVEC or PLANES (the column sums are taken from the fp32
 * n-direction B loads); M, N, R < 1, splitR outside 1..R, splitR > 1 without EPI_ATOMIC; C_hi / C_lo with EPI_ATOMIC or one
 * without the other; an operand missing or given where the problem does not read it; an address any table can reach outside its
 * arena (the K-major plane producers also read the r tables up to index 64 ceil(R / 64) - 8, and the MN-major ones 8 elements
 * from every 8-group start of aM / bN); a 16-byte fp32 load (r-, m- or n-direction 4-group), int4 table load, 16-byte plane
 * copy (8-group; 8 bytes per half under A_ALIGN4) or vector output store whose elements are not contiguous or whose address is
 * not aligned.  Arena lengths are element counts below 2^31.  Flag values beside B2G_GG_* above: */
#define B2G_GG_PLANES (1 << 6)
#define B2G_GG_A_ALIGN4 (1 << 7)
#define B2G_GG_MN_MAJOR (1 << 9)
#define B2G_GG_A_ROWLANES (1 << 14)
typedef struct {
  int64_t A, B, C, bias, mask, colsum;       /* offsets into f32; -1 = none (A and B are -1 under B2G_GG_PLANES) */
  int64_t aM, aR, bR, bN, cM, cN, kM, kN;    /* offsets into tabs; kM / kN -1 = cM / cN */
  int64_t bR_p, bN_p;                        /* offsets into tabs, K-major plane problems only; -1 = bR / bN */
  int64_t A_hi, A_lo, B_hi, B_lo;            /* offsets into u16, plane problems only; -1 = none */
  int64_t C_hi, C_lo;                        /* offsets into u16, -1 = none */
  int32_t M, N, R, flags, splitR;
} b2g_debug_gg_tc_problem;
int b2g_debug_gg_tc(int x3, const b2g_debug_gg_tc_problem* p, int n, float* f32, int64_t n_f32, uint16_t* u16, int64_t n_u16,
                    const int32_t* tabs, int64_t n_tabs);

/* Bring-up hook (not on the product path): one plane of one named device tensor of a SAC handle, copied to the host after the
 * handle's stream is synchronised.  BF16 planes come back as raw uint16 (elem_bytes 2), fp32 buffers as float (elem_bytes 4);
 * bytes must be numel * elem_bytes.  Returns B2G_EINVAL for an unknown name, a plane out of range or a size mismatch, and
 * B2G_ESTATE for an engine-v2 name (every BF16 name, and z0v) on a handle that does not run engine v2 (CNN policy, 64 x 64
 * image, 1 to 4 image channels, bf16x3).  The tensors hold what the LAST step left: read them right after the step, since
 * b2g_sac_act overwrites planes 0 and 1 of the policy's activations (S/obs, H1/pi .. F/pi).
 * <net> is pi, values or target; the backward tensors and natural weight planes exist for pi and values only.  B = batch,
 * Ci = image channels, Cp = 1 if Ci == 1 else 4, K1 = 64 Cp, KF = 576, FS = feature-row stride of the fp32 rows, H = hidden.
 *   S/obs, S/next_obs   3 planes  [B][16 Y][16 X][4 b][4 c][Cp]: normalised pixel (4Y + b, 4X + c) / 255; channels ci >= Ci zero
 *   H1/<net>            3 planes  [B][15][15][32]   conv1 output (NHWC, after ReLU)
 *   H2/<net>            3 planes  [B][6][6][64]     conv2 output
 *   H3/<net>            3 planes  [B][4][4][64]     conv3 output (= cnn_fc1 input row of 1024)
 *   F/<net>             3 planes  [B][KF]           512 cnn_fc1 features, the actuator value, the n_act actions (values only), zeros
 *   dz0pi / dz0v        2 planes  [B][H] / [B][3H]  fc0 pre-activation gradients (pi; vf | qf1 | qf2)
 *   dZ4/<net>           2 planes  [B][512]          cnn_fc1 output gradient, ReLU-masked
 *   dZ3/<net>           2 planes  [B][1024]         conv3 output gradient [B][4][4][64]
 *   dZ2/<net>           2 planes  [B][6][6][64]     conv2 output gradient
 *   dZ1                 2 planes  [B][15][15][2 nets][32]   conv1 output gradient of pi | values
 *   W1T/online          3 planes  [64 = pi | values][K1]   conv1 kernels transposed, K row of HWIO row r = conv1_krow(r, Ci)
 *   W1T/target          3 planes  [32][K1]                 (pad rows zero)
 *   W2T/<net>, W3T/<net>, WfT/<net>   3 planes  [N][K]: cnn2/w [64][512], cnn3/w [64][576], cnn_fc1/w [512][1024] transposed
 *   K0T/<net>           3 planes  [H or 3H = vf | qf1 | qf2][KF]   fc0 kernels transposed, rows padded with zeros to KF
 *   W2n/<net>, W3n/<net>, Wfn/<net>   2 planes  the HWIO / [in][out] kernels as stored: [512][64], [576][64], [1024][512]
 *   K0n/<net>           2 planes  [KF][H] (pi) / [KF][3H] (values: vf | qf1 | qf2), rows beyond each kernel's K zero
 *   F32/<net>           fp32      [B][FS]            the feature rows the head kernels read (columns as in F)
 *   z0/pi, z0/target    fp32      [B][H]             fc0 pre-activations without bias
 *   z0v                 fp32      [B][3H]            the same for vf | qf1 | qf2
 *   z0/vf, z0/qf1, z0/qf2  fp32   [B][H]             the same as separate buffers, on a handle WITHOUT engine v2 (B2G_ESTATE on
 *                                                    one with it: use z0v)
 *   rew_n, done_n       fp32      [B]                the reward and done the tail read (after the gather's normalisation and clip)
 *   a0/<head>, dz1/<head>  fp32   [B][H]             fc0 activations and fc1 pre-activation gradients; head = pi, vf, qf1, qf2
 *   dz0_pi / dz0_v3     fp32      [B][H] / [B][3H]   the fp32 values of dz0pi / dz0v */
int b2g_debug_tensor_info(const b2g_sac* h, const char* name, int64_t* numel, int32_t* planes, int32_t* elem_bytes);
int b2g_debug_tensor(b2g_sac* h, const char* name, int plane, void* dst, size_t bytes);

/* One named device buffer of a PPO2 / TRPO handle back to the host, after syncing the handle's stream, so that tests can hold
 * each actor-critic kernel to float64 of the inputs it read.  _info gives the element count and size (4: fp32, or int32 for
 * the row tables; 8: the int64 counters, and float64 for TRPO's part, amax, lspart and sc); bytes must be numel * elem_bytes.
 * B2G_EINVAL for an unknown name or a size mismatch.  The buffers hold what the LAST call left.  R = activation rows (PPO2:
 * max(minibatch, max(64, n_envs)); TRPO: max(N + 1, 64)), E = n_envs (TRPO 1), T = n_steps (TRPO N), XS = obs_dim rounded up
 * to 4, n_train / n_param = floats of the trained block / of the arena, D, A, H0, H1 as configured.
 * Both handles:
 *   P [n_param], G Mo Vo [n_train]     parameter arena (actor_critic.cuh order), gradient arena and Adam moments
 *   Z0 Y0 [R][2 H0], Y1 [R][2 H1]       layer-0 pre-activations (no bias) and both layers' tanh outputs: pi | vf columns
 *   r_obs [T + 1][E][XS], r_act [T + 1][E][A], r_val r_nlp r_done [T + 1][E], r_rew r_adv r_ret [T][E], lastv [E]
 *   a_out [R][A], a_v a_nlp [R]         the actor's predict outputs; act_rowoff int32 [E]; counters int64 [4]
 * PPO2 (M = minibatch, NP = noptepochs * n_batch):
 *   sz sdm sdls [R][A], sv snlp sadv sdv [R], dZ1 [R][2 H1], dZ0 [R][2 H0]   the tail's scratch and outputs
 *   part [128] (norm partials), met [16], hp [4], rowidx rowoff perm int32 [NP]
 * TRPO (NF = ceil(N / 5), V = 128, K = 10 line-search candidates):
 *   atarg nlp_old [N], mu_old sdm sdls [N][A], u [NF][A], T0 [NF][H0], T1 [NF][H1], dZ1 [R][H1], dZ0 [R][H0]
 *   X Rv Pv Zv FS Gv [n_train]          CG vectors, the full step and the value gradient, in the arena layout
 *   part amax [128], lspart [K][64][2], sc [16] (float64), met [16]
 *   cand [K][H0 + H0 H1 + H1 + H1 A + 2 A] (b0, W1, b1, pi/w, pi/b, logstd blocks of all K, block after block)
 *   Y0c [K][N][H0], Y1c [K][N][H1], dZls [N][H0], vZ0 vY0 vdZ0 [V][H0], vY1 vdZ1 [V][H1], perm vrowoff int32 [max(1, vf_iters N)] */
int b2g_debug_ppo_tensor_info(const b2g_ppo* h, const char* name, int64_t* numel, int32_t* elem_bytes);
int b2g_debug_ppo_tensor(b2g_ppo* h, const char* name, void* dst, size_t bytes);
int b2g_debug_trpo_tensor_info(const b2g_trpo* h, const char* name, int64_t* numel, int32_t* elem_bytes);
int b2g_debug_trpo_tensor(b2g_trpo* h, const char* name, void* dst, size_t bytes);
/* The policy gradient of b2g_trpo_step_explicit on obs [N, obs_dim], actions [N, n_actions] and raw advantages [N], then
 * `iters` (1..64) conjugate-gradient iterations and nothing after them.  prev [3 n_train + 2 * SC_N(16)] receives x, r and p
 * (arena layout) and the 16 float64 CG scalars as they stood before the last iteration; the debug tensors then hold that
 * iteration's z = F p_prev (Zv), x, r, p after its p update (X, Rv, Pv) and scalars (sc). */
int b2g_debug_trpo_cg(b2g_trpo* h, const float* obs, const float* actions, const float* adv, int iters, float* prev);

#ifdef __cplusplus
}
#endif
#endif /* B200GRASP_H_ */
