// group.cu — a volume group: the static map and a pool of car-volume slots on one GPU, and DynSLAM's whole multi-volume frame
// (instance frames cut out, every car fused, the static map fused, the layers composited) as one enqueue.
//
// Every slot is created up front with its engine, scene, render state and images, so the device waits of b200_engine_create
// and the cudaFree calls of b200_engine_destroy happen at b200_group_create / b200_group_destroy only. A new car track takes a
// free slot and restarts it on the device (b200_volume_restart_async): no host wait, no allocation. The frame is the sequence
// the engine handle documents in include/b200fusion.h, built from the same calls and launchers, so its bytes are the bytes of
// that sequence. The silhouette ops and the composite layers reach the device as launch parameters (copied when the kernel is
// enqueued, held by value in a captured graph), so no host buffer of the caller has to outlive the call.
#include "engine.h"

#include <cstdio>
#include <cstring>
#include <vector>

struct GroupSlot {
  b200_engine *e;
  b200_scene scene;
  b200_render_state rs;
  b200_group_images img;
  void *arena;               // one allocation: scene, render state and images of the slot
  bool started;              // b200_group_track_start has run on it
  bool needJoin;             // work enqueued on its stream that the origin stream has not waited for yet
};

struct b200_group {
  b200_engine *se;           // the caller's static engine, scene and render state
  b200_scene *ss;
  b200_render_state *srs;
  b200_vec4f *sPoints, *sNormals;
  int maxCars, w, h;
  float dimFactor, tintStrength;
  std::vector<GroupSlot> slots;
  std::vector<b200_silhouette_op> ops;       // host scratch of one frame, sized at create
  std::vector<b200_instance_layer> layers;
  std::vector<unsigned char> seen;
  char err[512];
};

#define GCK(call)                                                                                  \
  do {                                                                                             \
    cudaError_t _e = (call);                                                                       \
    if (_e != cudaSuccess) {                                                                       \
      snprintf(g->err, sizeof(g->err), "%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(_e)); \
      return B200_ERR_CUDA;                                                                        \
    }                                                                                              \
  } while (0)

// an engine call's failure, with the engine's own message
#define GENG(eng, call)                                                                            \
  do {                                                                                             \
    const b200_status _s = (call);                                                                 \
    if (_s != B200_OK) { snprintf(g->err, sizeof(g->err), "%.500s", b200_last_error(eng)); return _s; }   \
  } while (0)

static thread_local char g_groupCreateErr[512] = "";

static size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

// the slot's buffers carved out of one allocation, in the order below
static b200_status slot_alloc(b200_group *g, GroupSlot &sl, const b200_group_config *cfg) {
  const size_t px = (size_t)g->w * g->h, noTotal = (size_t)cfg->numBuckets + cfg->excessSize;
  const size_t sizes[] = {
      (size_t)cfg->numBlocks * B200_SDF_BLOCK_SIZE3 * sizeof(b200_voxel), (size_t)cfg->numBlocks * sizeof(int32_t),
      noTotal * sizeof(b200_hash_entry), (size_t)cfg->excessSize * sizeof(int32_t),
      (size_t)cfg->numBlocks * sizeof(b200_vec3i), noTotal, px * sizeof(b200_vec2f), px * sizeof(b200_vec4f), px * sizeof(b200_vec4u),
      px * sizeof(b200_vec4u), px * sizeof(float), px * sizeof(b200_vec4u), px * sizeof(float), px * sizeof(b200_vec4f),
      px * sizeof(b200_vec4f)};
  const int n = (int)(sizeof(sizes) / sizeof(sizes[0]));
  size_t total = 0;
  for (int i = 0; i < n; ++i) total += align256(sizes[i]);
  GCK(cudaMalloc(&sl.arena, total));
  uint8_t *p[sizeof(sizes) / sizeof(sizes[0])];
  size_t off = 0;
  for (int i = 0; i < n; ++i) { p[i] = (uint8_t *)sl.arena + off; off += align256(sizes[i]); }
  b200_scene &s = sl.scene;
  memset(&s, 0, sizeof(s));
  s.d_voxels = (b200_voxel *)p[0]; s.d_allocationList = (int32_t *)p[1]; s.d_hash = (b200_hash_entry *)p[2];
  s.d_excessList = (int32_t *)p[3]; s.d_swapStates = nullptr;
  s.numBlocks = cfg->numBlocks; s.numBuckets = cfg->numBuckets; s.excessSize = cfg->excessSize;
  s.lastFreeBlockId = cfg->numBlocks - 1; s.lastFreeExcessListId = cfg->excessSize - 1;
  s.voxelSize = cfg->voxelSize; s.mu = cfg->mu; s.maxW = cfg->maxW;
  s.viewFrustum_min = g->ss->viewFrustum_min; s.viewFrustum_max = g->ss->viewFrustum_max;
  s.stopIntegratingAtMaxW = g->ss->stopIntegratingAtMaxW; s.useSwapping = 0;
  b200_render_state &r = sl.rs;
  memset(&r, 0, sizeof(r));
  r.d_visibleBlockPositions = (b200_vec3i *)p[4]; r.d_entriesVisibleType = p[5]; r.d_minmax = (b200_vec2f *)p[6];
  r.d_raycastResult = (b200_vec4f *)p[7]; r.d_raycastImage = (b200_vec4u *)p[8];
  r.img_w = g->w; r.img_h = g->h;
  b200_group_images &im = sl.img;
  im.d_instance_rgb = (b200_vec4u *)p[9]; im.d_instance_depth = (float *)p[10];
  im.d_colour_render = (b200_vec4u *)p[11]; im.d_depth_render = (float *)p[12];
  im.d_points = (b200_vec4f *)p[13]; im.d_normals = (b200_vec4f *)p[14];
  return B200_OK;
}

extern "C" {

void b200_group_destroy(b200_group *g) {
  if (!g) return;
  for (GroupSlot &sl : g->slots) {
    b200_engine_destroy(sl.e);           // waits for the slot's stream first
    if (sl.arena) cudaFree(sl.arena);
  }
  cudaGetLastError();
  delete g;
}

const char *b200_group_last_error(const b200_group *g) { return g ? g->err : g_groupCreateErr; }

static b200_status group_create_body(const b200_group_config *cfg_in, b200_group *g) {
  b200_group_config c = *cfg_in;
  if (c.numBlocks <= 0) c.numBlocks = 7142;
  if (c.numBuckets <= 0) c.numBuckets = 0x100000;
  if (c.excessSize <= 0) c.excessSize = 0x80000;
  if (c.voxelSize <= 0.0f) c.voxelSize = 0.035f;
  if (c.mu <= 0.0f) c.mu = 1.0f;
  if (c.maxW <= 0) c.maxW = 50;
  g->se = c.static_engine; g->ss = c.static_scene; g->srs = c.static_rs;
  g->sPoints = c.static_points; g->sNormals = c.static_normals;
  g->w = c.img_w > 0 ? c.img_w : c.static_rs->img_w;
  g->h = c.img_h > 0 ? c.img_h : c.static_rs->img_h;
  g->maxCars = c.max_cars; g->dimFactor = c.dim_factor; g->tintStrength = c.tint_strength;
  if (g->w != c.static_rs->img_w || g->h != c.static_rs->img_h) {
    snprintf(g->err, sizeof(g->err), "group_create: the car image size %dx%d differs from the static render state's %dx%d", g->w, g->h,
             c.static_rs->img_w, c.static_rs->img_h);
    return B200_ERR_INVALID;
  }
  const int device = g->se->device;
  GCK(cudaSetDevice(device));
  g->slots.resize((size_t)c.max_cars);
  memset(g->slots.data(), 0, sizeof(GroupSlot) * g->slots.size());
  g->ops.resize((size_t)c.max_cars * 2 + 1);
  g->layers.resize((size_t)c.max_cars + 1);
  g->seen.resize((size_t)c.max_cars);
  for (int i = 0; i < c.max_cars; ++i) {
    GroupSlot &sl = g->slots[(size_t)i];
    b200_engine_config ec{};
    ec.device = device; ec.numBlocks = c.numBlocks; ec.numBuckets = c.numBuckets; ec.excessSize = c.excessSize;
    ec.img_w = g->w; ec.img_h = g->h; ec.decayRingItems = c.decayRingItems;
    ec.stream = c.shared_stream ? b200_engine_stream(g->se) : nullptr;
    b200_status st = b200_engine_create(&ec, &sl.e);
    if (st) { snprintf(g->err, sizeof(g->err), "group_create: slot %d: %.480s", i, b200_last_error(nullptr)); return st; }
    st = slot_alloc(g, sl, &c); if (st) return st;
    // the event and counters b200_engine_wait_engine uses, made here rather than inside the first frame
    GENG(sl.e, b200_engine_wait_engine(sl.e, g->se));
    GENG(g->se, b200_engine_wait_engine(g->se, sl.e));
  }
  GCK(cudaDeviceSynchronize());
  return B200_OK;
}

b200_status b200_group_create(const b200_group_config *cfg, b200_group **out) {
  if (out) *out = nullptr;
  if (!cfg || !out || !cfg->static_engine || !cfg->static_scene || !cfg->static_rs || !cfg->static_points || !cfg->static_normals ||
      cfg->max_cars < 0) {
    snprintf(g_groupCreateErr, sizeof(g_groupCreateErr), "group_create: null configuration, output, static volume or ICP buffers, or max_cars < 0");
    return B200_ERR_INVALID;
  }
  b200_group *g = new b200_group();
  const b200_status st = group_create_body(cfg, g);
  if (st) {                 // nothing stays allocated after a failed create; the reason survives in b200_group_last_error(NULL)
    snprintf(g_groupCreateErr, sizeof(g_groupCreateErr), "%s", g->err);
    b200_group_destroy(g);
    return st;
  }
  *out = g;
  return B200_OK;
}

b200_status b200_group_slot(b200_group *g, int slot, b200_engine **engine, b200_scene **scene, b200_render_state **rs) {
  if (!g) return B200_ERR_INVALID;
  if (slot < 0 || slot >= g->maxCars) { snprintf(g->err, sizeof(g->err), "slot %d out of range [0, %d)", slot, g->maxCars); return B200_ERR_INVALID; }
  GroupSlot &sl = g->slots[(size_t)slot];
  if (engine) *engine = sl.e;
  if (scene) *scene = &sl.scene;
  if (rs) *rs = &sl.rs;
  return B200_OK;
}

b200_status b200_group_slot_images(b200_group *g, int slot, b200_group_images *out) {
  if (!g) return B200_ERR_INVALID;
  if (slot < 0 || slot >= g->maxCars || !out) { snprintf(g->err, sizeof(g->err), "slot %d out of range [0, %d) or no output", slot, g->maxCars); return B200_ERR_INVALID; }
  *out = g->slots[(size_t)slot].img;
  return B200_OK;
}

b200_status b200_group_track_start(b200_group *g, int slot) {
  if (!g) return B200_ERR_INVALID;
  if (slot < 0 || slot >= g->maxCars) { snprintf(g->err, sizeof(g->err), "slot %d out of range [0, %d)", slot, g->maxCars); return B200_ERR_INVALID; }
  GroupSlot &sl = g->slots[(size_t)slot];
  // behind everything the group has enqueued so far, so that the restart joins a capture begun on the origin stream
  GENG(sl.e, b200_engine_wait_engine(sl.e, g->se));
  GENG(sl.e, b200_volume_restart_async(sl.e, &sl.scene, &sl.rs));
  sl.started = true;
  sl.needJoin = true;
  return B200_OK;
}

static bool mask_missing(const b200_mask &m) { return m.d_data == nullptr; }

b200_status b200_group_frame_async(b200_group *g, b200_vec4u *d_rgb, float *d_depth, const b200_view *static_view, const b200_group_car *cars,
                                   int n, const int32_t *decay, b200_vec4u *d_out_color, float *d_out_depth) {
  if (!g) return B200_ERR_INVALID;
#define REJECT(...) do { snprintf(g->err, sizeof(g->err), "group_frame: " __VA_ARGS__); return B200_ERR_INVALID; } while (0)
  // every rejection before anything is enqueued
  if (!d_rgb || !d_depth || !static_view || !d_out_color || !d_out_depth || n < 0 || (n > 0 && !cars)) REJECT("null argument or n < 0");
  if (n > g->maxCars) REJECT("%d cars, the group has %d slots", n, g->maxCars);
  if (static_view->depth_w != g->w || static_view->depth_h != g->h || static_view->rgb_w != g->w || static_view->rgb_h != g->h)
    REJECT("the static view is %dx%d (colour %dx%d), the group's frames %dx%d", static_view->depth_w, static_view->depth_h,
           static_view->rgb_w, static_view->rgb_h, g->w, g->h);
  memset(g->seen.data(), 0, g->seen.size());
  for (int k = 0; k < n; ++k) {
    const b200_group_car &c = cars[k];
    if (c.slot < 0 || c.slot >= g->maxCars) REJECT("car %d: slot %d out of range [0, %d)", k, c.slot, g->maxCars);
    if (g->seen[(size_t)c.slot]) REJECT("car %d: slot %d appears twice", k, c.slot);
    g->seen[(size_t)c.slot] = 1;
    if (!g->slots[(size_t)c.slot].started) REJECT("car %d: slot %d was never started (b200_group_track_start)", k, c.slot);
    if (c.action < 0 || c.action > 2) REJECT("car %d: unknown action %d", k, c.action);
    if (c.action == 2 && mask_missing(c.copy_mask)) REJECT("car %d: copy mask missing", k);
    if (c.action != 0 && mask_missing(c.delete_mask)) REJECT("car %d: delete mask missing", k);
  }
#undef REJECT
  GCK(cudaSetDevice(g->se->device));
  // 1. the silhouettes, in the given order, each extracted car into its slot's instance frame. A fused car without an extract
  //    fuses an empty instance frame (white, depth 0): an extract with empty boxes writes exactly that and blanks nothing.
  int nOps = 0;
  for (int k = 0; k < n; ++k) {
    const b200_group_car &c = cars[k];
    if (c.action == 0) continue;
    b200_silhouette_op &o = g->ops[(size_t)nOps++];
    memset(&o, 0, sizeof(o));
    o.action = c.action; o.copy_mask = c.copy_mask; o.delete_mask = c.delete_mask;
    o.d_dest_rgb = g->slots[(size_t)c.slot].img.d_instance_rgb; o.d_dest_depth = g->slots[(size_t)c.slot].img.d_instance_depth;
  }
  for (int k = 0; k < n; ++k) {
    const b200_group_car &c = cars[k];
    if (c.action == 2 || !c.fuse) continue;
    b200_silhouette_op &o = g->ops[(size_t)nOps++];
    memset(&o, 0, sizeof(o));
    o.action = 2;
    o.copy_mask.x0 = o.delete_mask.x0 = 0; o.copy_mask.x1 = o.delete_mask.x1 = -1;   // no pixel lies in an empty box
    o.d_dest_rgb = g->slots[(size_t)c.slot].img.d_instance_rgb; o.d_dest_depth = g->slots[(size_t)c.slot].img.d_instance_depth;
  }
  if (nOps > 0) launch_process_silhouettes(g->se, d_rgb, d_depth, g->w, g->h, g->ops.data(), nOps);
  GCK(cudaGetLastError());
  // 2. every fused car: its stream waits for the silhouettes, then its volume's frame with the colour and depth renders
  b200_frame_opts o{};
  o.doRaycast = 1;
  if (decay) { o.doDecay = 1; o.decayMaxWeight = decay[0]; o.decayMinAge = decay[1]; }
  int nLayers = 0;
  for (int k = 0; k < n; ++k) {
    const b200_group_car &c = cars[k];
    if (!c.fuse) continue;
    GroupSlot &sl = g->slots[(size_t)c.slot];
    GENG(sl.e, b200_engine_wait_engine(sl.e, g->se));
    b200_view v{};
    v.d_depth = sl.img.d_instance_depth; v.d_rgb = sl.img.d_instance_rgb;
    v.depth_w = v.rgb_w = g->w; v.depth_h = v.rgb_h = g->h;
    memcpy(v.M_d, c.cam.M, sizeof(v.M_d)); memcpy(v.invM_d, c.cam.invM, sizeof(v.invM_d)); memcpy(v.M_rgb, c.cam.M, sizeof(v.M_rgb));
    memcpy(v.proj_d, c.cam.proj, sizeof(v.proj_d)); memcpy(v.proj_rgb, c.cam.proj, sizeof(v.proj_rgb));
    v.depthWeighting = 0; v.requiresFullRendering = 1;
    b200_frame_opts co = o;
    co.d_colourRender = sl.img.d_colour_render; co.d_depthRender = sl.img.d_depth_render;
    GENG(sl.e, b200_process_frame_async(sl.e, &sl.scene, &sl.rs, &v, sl.img.d_points, sl.img.d_normals, &co));
    sl.needJoin = true;
    b200_instance_layer &l = g->layers[(size_t)nLayers++];
    l.d_color = sl.img.d_colour_render; l.d_depth = sl.img.d_depth_render;
    memcpy(l.tint, c.tint, sizeof(l.tint));
  }
  // 3. the static map, its depth render straight into the output depth
  b200_frame_opts so = o;
  so.d_depthRender = d_out_depth;
  GENG(g->se, b200_process_frame_async(g->se, g->ss, g->srs, static_view, g->sPoints, g->sNormals, &so));
  // 4. the joins: the origin stream waits for every slot it has not waited for yet
  for (GroupSlot &sl : g->slots) {
    if (!sl.needJoin) continue;
    GENG(g->se, b200_engine_wait_engine(g->se, sl.e));
    sl.needJoin = false;
  }
  // 5. the static layer (its shaded raycast image, written by the ICP pass, and its depth render) under the cars' layers, read in
  //    place as the background of one compositing pass
  const int px = g->w * g->h;
  launch_composite_layers(g->se, d_out_color, d_out_depth, px, g->layers.data(), nLayers, g->dimFactor >= 0.0f, g->dimFactor,
                          g->tintStrength, nullptr, g->srs->d_raycastImage, d_out_depth);
  GCK(cudaGetLastError());
  return B200_OK;
}

b200_status b200_group_sync(b200_group *g) {
  if (!g) return B200_ERR_INVALID;
  GENG(g->se, b200_sync(g->se, g->ss, g->srs));
  for (GroupSlot &sl : g->slots) GENG(sl.e, b200_sync(sl.e, &sl.scene, &sl.rs));
  return B200_OK;
}

}  // extern "C"
