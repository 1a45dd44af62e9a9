/*
 * b200fusion_diag.h — measurement and test hooks of libb200fusion. NOT part of the drop-in boundary
 * (include/b200fusion.h): nothing on the reference side binds these. bench.py reads the timers and the
 * launch trace, tests/ call the self-test and lower the rendering-block cap.
 */
#ifndef B200FUSION_DIAG_H
#define B200FUSION_DIAG_H
#include "b200fusion.h"
#ifdef __cplusplus
extern "C" {
#endif

typedef struct {
  float ms_allocate, ms_integrate, ms_expected, ms_raycast, ms_decay, ms_total;
  int64_t launches;            /* kernels launched by this engine since creation */
  int32_t noVisibleBlocks, noIntegratedBlocks;
  /* timing mode 2: CUDA-event pairs around EVERY IntegrateIntoScene launch since the mode was set */
  float ring_ms_integrate;     /* sum of the launch durations */
  int32_t ring_count;          /* number of launches measured */
  int64_t totalIntegratedBlocks; /* cumulative blocks integrated since engine creation */
  int64_t droppedSnapshots;    /* decay-queue snapshots dropped because the queue or the ring was full (b200_engine_config) */
} b200_frame_stats;

/* 0 = off; 1 = per-stage CUDA events of the last fused frame; 2 = 1 + an event pair around every
   integrate launch (ring of 8192 frames), reset whenever the mode is set; 3 = an event pair around EVERY
   kernel launch of the frame path (launch trace, read and cleared by b200_get_trace; perturbs the timing) */
void b200_set_timing(b200_engine *e, int enabled);
/* "kernel start_us end_us" lines (relative to the first traced launch); returns the number of bytes written */
int b200_get_trace(b200_engine *e, char *out, int cap);
b200_status b200_get_stats(b200_engine *e, b200_frame_stats *out);

/* Self-test of the division sequences of the default IntegrateIntoScene kernel (integrate.cu, variant V3): on the
   engine's device, `pairs` pseudo-random operand pairs (a, b) drawn from the ranges the kernel's fast path accepts
   (|a| in {0} U [2^-40, 2^40], b in [2^-20, 2^20], plus the constant divisors mu, 255, 32767 and the integer weights
   1..271) are divided with the kernel's sequence and with the IEEE operator `/` (what DA/ITMSceneReconstructionEngine.h
   :14-128 evaluates on the host); *mismatches receives the number of quotients whose bits differ (signed zeros
   compare equal). Test infrastructure only. */
b200_status b200_selftest_divide(b200_engine *e, uint64_t pairs, uint64_t seed, float mu, uint64_t *mismatches);


/* MAX_RENDERING_BLOCKS (DeviceAgnostic/ITMVisualisationEngine.h:25) of this engine; tests lower it to reach the cap rule
   (Vis_CUDA.cu:609) with small scenes. n <= 0 restores the reference's constant. */
void b200_diag_set_max_rendering_blocks(b200_engine *e, int n);

/* The IntegrateIntoScene kernel that this engine's last integrate launch ran, and its grid (CTAs): 0 = LDG, 1 = TMA, 2 = V3,
   3 = V4 with two voxels per lane, 4 = V4 with four voxels per lane; + 8 in tolerance mode (B200_INTEGRATE_IMPL=fast).
   -1 and 0 before the first launch. Tests use it to check that the variant they mean to exercise really ran. */
void b200_diag_last_integrate(const b200_engine *e, int *kernel, int *grid);

/* Seed the decay queue the way AllocateSceneFromDepth does (Reco_CUDA.cu:302-316), without an allocation: the n block
   positions at d_positions (device memory, 0 <= n <= numBlocks) become the newest snapshot, through the same snapshot ring
   and queue bookkeeping. frameIdx is not advanced; b200_diag_set_frame_index sets it (the `currentFrame` that Decay
   measures block ages against). Tests use both to hand the engine exactly the decay state they hand the oracle. */
b200_status b200_diag_push_decay_snapshot(b200_engine *e, const b200_vec3i *d_positions, int n);
void b200_diag_set_frame_index(b200_engine *e, int32_t f);

/* While the launch trace is on (b200_set_timing(e, 3)) a few CTAs of the allocation's list pass stamp %globaltimer at their
   phase boundaries (8 stamps x 4 CTAs, nanoseconds); copies up to 64 of them out. Measurement only. */
int b200_diag_read_debug(b200_engine *e, unsigned long long *out, int n);

#ifdef __cplusplus
}
#endif
#endif /* B200FUSION_DIAG_H */
