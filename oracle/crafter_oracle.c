/*
 * ORACLE (test infrastructure, never shipped, never imported by crafter_b200/):
 * single-environment CPU restatement of the reference hot path danijar/crafter
 * `Env.reset / Env.step / Env.render` under the keyed-random contract of oracle/keyed_rng.py.
 * Each function cites the reference file:line it follows (paths relative to /root/reference).
 *
 * Pinned against the unmodified reference run in the build container: tools/make_golden.py
 * dumps trajectories from oracle/ref_harness.py into tests/golden/, tests/test_oracle_golden.py
 * replays them here bit for bit (grid, slots, inventory, achievements, vitals, reward, done, obs).
 * Noise arithmetic (oracle/opensimplex_ref.c) is the one UNPINNED piece -- see its header.
 *
 * Style: deliberately reference-shaped (one struct per object, append-only slot list, full scans)
 * so that it stays an independent statement from the SoA / fixed-capacity CUDA kernels.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

void osn_init(int64_t seed, int16_t *perm, int16_t *perm_grad_index3);
double osn_noise3(const int16_t *perm, const int16_t *pgi, double x, double y, double z);

/* ---- rule tables: crafter/data.yaml --------------------------------------------------------- */
enum { /* data.yaml:20-32, ids as engine.py:29-30 (0 = None) */
  M_NONE = 0, M_WATER, M_GRASS, M_STONE, M_PATH, M_SAND, M_TREE, M_LAVA, M_COAL, M_IRON,
  M_DIAMOND, M_TABLE, M_FURNACE };
enum { /* data.yaml:39-55 */
  I_HEALTH = 0, I_FOOD, I_DRINK, I_ENERGY, I_SAPLING, I_WOOD, I_STONE, I_COAL, I_IRON, I_DIAMOND,
  I_WOOD_PICKAXE, I_STONE_PICKAXE, I_IRON_PICKAXE, I_WOOD_SWORD, I_STONE_SWORD, I_IRON_SWORD,
  N_ITEMS };
enum { /* data.yaml:80-102 */
  A_COLLECT_COAL = 0, A_COLLECT_DIAMOND, A_COLLECT_DRINK, A_COLLECT_IRON, A_COLLECT_SAPLING,
  A_COLLECT_STONE, A_COLLECT_WOOD, A_DEFEAT_SKELETON, A_DEFEAT_ZOMBIE, A_EAT_COW, A_EAT_PLANT,
  A_MAKE_IRON_PICKAXE, A_MAKE_IRON_SWORD, A_MAKE_STONE_PICKAXE, A_MAKE_STONE_SWORD,
  A_MAKE_WOOD_PICKAXE, A_MAKE_WOOD_SWORD, A_PLACE_FURNACE, A_PLACE_PLANT, A_PLACE_STONE,
  A_PLACE_TABLE, A_WAKE_UP, N_ACH };
enum { /* data.yaml:1-18 */
  ACT_NOOP = 0, ACT_LEFT, ACT_RIGHT, ACT_UP, ACT_DOWN, ACT_DO, ACT_SLEEP, ACT_PLACE_STONE,
  ACT_PLACE_TABLE, ACT_PLACE_FURNACE, ACT_PLACE_PLANT, ACT_MAKE_WOOD_PICKAXE,
  ACT_MAKE_STONE_PICKAXE, ACT_MAKE_IRON_PICKAXE, ACT_MAKE_WOOD_SWORD, ACT_MAKE_STONE_SWORD,
  ACT_MAKE_IRON_SWORD };
enum { T_PLAYER = 1, T_COW, T_ZOMBIE, T_SKELETON, T_ARROW, T_PLANT };
enum { D_SEED = 0, D_WG_MAT, D_WG_OBJ, D_UPDATE, D_BALANCE, D_NOISE };

static const int DIRS[4][2] = {{-1, 0}, {1, 0}, {0, -1}, {0, 1}}; /* objects.py:33-34 */

typedef struct { int8_t mat, req_item, recv_item, recv_ach, leaves; double prob; } CollectRule;
static const CollectRule COLLECT[] = { /* data.yaml:57-64 */
    {M_TREE, -1, I_WOOD, A_COLLECT_WOOD, M_GRASS, 1.0},
    {M_STONE, I_WOOD_PICKAXE, I_STONE, A_COLLECT_STONE, M_PATH, 1.0},
    {M_COAL, I_WOOD_PICKAXE, I_COAL, A_COLLECT_COAL, M_PATH, 1.0},
    {M_IRON, I_STONE_PICKAXE, I_IRON, A_COLLECT_IRON, M_PATH, 1.0},
    {M_DIAMOND, I_IRON_PICKAXE, I_DIAMOND, A_COLLECT_DIAMOND, M_PATH, 1.0},
    {M_WATER, -1, I_DRINK, A_COLLECT_DRINK, M_WATER, 1.0},
    {M_GRASS, -1, I_SAPLING, A_COLLECT_SAPLING, M_GRASS, 0.1},
};
typedef struct { int8_t item, amount, result_mat, ach; uint16_t where; } PlaceRule;
#define MB(m) (1u << (m))
static const PlaceRule PLACE[4] = { /* data.yaml:66-70, order = actions 7..10 */
    {I_STONE, 1, M_STONE, A_PLACE_STONE, MB(M_GRASS) | MB(M_SAND) | MB(M_PATH) | MB(M_WATER) | MB(M_LAVA)},
    {I_WOOD, 2, M_TABLE, A_PLACE_TABLE, MB(M_GRASS) | MB(M_SAND) | MB(M_PATH)},
    {I_STONE, 4, M_FURNACE, A_PLACE_FURNACE, MB(M_GRASS) | MB(M_SAND) | MB(M_PATH)},
    {I_SAPLING, 1, -1 /* object: Plant */, A_PLACE_PLANT, MB(M_GRASS)},
};
typedef struct { int8_t wood, stone, coal, iron, need_furnace, gives, ach; } MakeRule;
static const MakeRule MAKE[6] = { /* data.yaml:72-78, order = actions 11..16 */
    {1, 0, 0, 0, 0, I_WOOD_PICKAXE, A_MAKE_WOOD_PICKAXE},
    {1, 1, 0, 0, 0, I_STONE_PICKAXE, A_MAKE_STONE_PICKAXE},
    {1, 0, 1, 1, 1, I_IRON_PICKAXE, A_MAKE_IRON_PICKAXE},
    {1, 0, 0, 0, 0, I_WOOD_SWORD, A_MAKE_WOOD_SWORD},
    {1, 1, 0, 0, 0, I_STONE_SWORD, A_MAKE_STONE_SWORD},
    {1, 0, 1, 1, 1, I_IRON_SWORD, A_MAKE_IRON_SWORD},
};
#define WALKABLE (MB(M_GRASS) | MB(M_SAND) | MB(M_PATH))            /* data.yaml:34-37 */
#define WALKABLE_PLAYER (WALKABLE | MB(M_LAVA))                     /* objects.py:95-97 */
#define WALKABLE_ARROW (WALKABLE | MB(M_WATER) | MB(M_LAVA))        /* objects.py:369-371 */

/* ---- keyed random contract (oracle/keyed_rng.py) ------------------------------------------- */
static void philox(uint32_t k0, uint32_t k1, uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                   uint32_t out[4]) {
  for (int r = 0; r < 10; ++r) {
    uint64_t p0 = (uint64_t)0xD2511F53u * c0, p1 = (uint64_t)0xCD9E8D57u * c2;
    uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0, n1 = (uint32_t)p1;
    uint32_t n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1, n3 = (uint32_t)p0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

typedef struct { uint32_t seed, domain, k, c1, c2, c3; long draws; } Rng;
static void rng_ctx(Rng *r, uint32_t domain, uint32_t c1, uint32_t c2, uint32_t c3) {
  r->domain = domain; r->k = 0; r->c1 = c1; r->c2 = c2; r->c3 = c3;
}
static double rng_uniform(Rng *r) {
  uint32_t w[4];
  philox(r->seed, r->domain, r->k++, r->c1, r->c2, r->c3, w);
  r->draws++;
  return (double)((((uint64_t)w[1] << 32) | w[0]) >> 11) * (1.0 / 9007199254740992.0);
}
static uint32_t rng_randint(Rng *r, uint32_t n) {
  uint32_t w[4];
  philox(r->seed, r->domain, r->k++, r->c1, r->c2, r->c3, w);
  r->draws++;
  return (uint32_t)(((uint64_t)w[0] * n) >> 32);
}

/* CPython >= 3.8 tuple hash of two small non-negative ints, then % (2**31 - 1):
 * env.py:74 `hash((self._seed, self._episode)) % (2 ** 31 - 1)`. */
int64_t co_world_seed(int64_t seed, int64_t episode) {
  const uint64_t P1 = 11400714785074694791ULL, P2 = 14029467366897019727ULL,
                 P5 = 2870177450012600261ULL;
  uint64_t acc = P5, lanes[2] = {(uint64_t)seed, (uint64_t)episode};
  for (int i = 0; i < 2; ++i) {
    acc += lanes[i] * P2;
    acc = (acc << 31) | (acc >> 33);
    acc *= P1;
  }
  acc += 2ULL ^ (P5 ^ 3527539ULL);
  if (acc == (uint64_t)-1) acc = 1546275796ULL;
  int64_t h = (int64_t)acc, m = 2147483647LL, r = h % m;
  if (r < 0) r += m; /* Python floored modulo */
  return r;
}

/* ---- world: crafter/engine.py:24-117 -------------------------------------------------------- */
typedef struct {
  int type, x, y, health, removed;
  int facing;   /* Player, Arrow: index into DIRS */
  int cooldown; /* Zombie objects.py:288 */
  int reload;   /* Skeleton objects.py:321 */
  int grown;    /* Plant objects.py:392 */
} Obj;

typedef struct {
  int ux, uy, iw, ih, dw, dh; /* unit, item icon, digit sizes */
  int item_pos[N_ITEMS][2], digit_pos[N_ITEMS][2];
  uint8_t *mat_tex;   /* [13][ux][uy][3] */
  uint8_t *obj_tex;   /* [14][ux][uy][4] */
  uint8_t *item_tex;  /* [16][iw][ih][4] */
  uint8_t *digit_tex; /* [10][dw][dh][4] */
  double *vignette;   /* [gx*ux][gy*uy] engine.py:213-218, computed by numpy on the host */
} Tex;

typedef struct CoEnv {
  int aw, ah, vw, vh, sw, sh, length, reward_flag;
  int gx, gy, item_rows; /* local grid env.py:42-44 */
  int ncx, ncy;
  int64_t seed, episode;
  int step;
  double daylight;
  const double *daylight_table; /* [length+2], env.py:135-139 evaluated by numpy on the host */
  int n_daylight;
  Rng rng;
  uint8_t *mat;     /* [aw][ah] engine.py:38 */
  int32_t *obj_map; /* [aw][ah] slot index, 0 = empty engine.py:39 */
  uint8_t *tunnels;
  uint8_t *touched; /* chunk ever held an object: engine.py:36,57,79 */
  Obj *objs; int n_slots, cap_slots; /* slot 0 unused engine.py:37 */
  /* player state objects.py:70-82 */
  int inventory[N_ITEMS], achievements[N_ACH];
  int action, sleeping, p_last_health, hunger2, thirst2, fatigue, recover2;
  int last_health; uint32_t unlocked; /* env.py:53-54 */
  int16_t perm[256], pgi[256];
  Tex tex;
} CoEnv;

#define CELL(e, x, y) ((x) * (e)->ah + (y))
static int inside(const CoEnv *e, int x, int y) { /* engine.py:267-268 */
  return x >= 0 && x < e->aw && y >= 0 && y < e->ah;
}
static int chunk_of(const CoEnv *e, int x, int y) { return (x / 12) * e->ncy + (y / 12); }

static int world_add(CoEnv *e, Obj o) { /* engine.py:50-57 */
  if (e->n_slots == e->cap_slots) {
    e->cap_slots *= 2;
    e->objs = (Obj *)realloc(e->objs, sizeof(Obj) * e->cap_slots);
  }
  int idx = e->n_slots++;
  o.removed = 0;
  e->objs[idx] = o;
  e->obj_map[CELL(e, o.x, o.y)] = idx;
  e->touched[chunk_of(e, o.x, o.y)] = 1;
  return idx;
}
static void world_remove(CoEnv *e, int idx) { /* engine.py:59-65 */
  Obj *o = &e->objs[idx];
  if (o->removed) return;
  e->obj_map[CELL(e, o->x, o->y)] = 0;
  o->removed = 1;
}
static void world_move(CoEnv *e, int idx, int x, int y) { /* engine.py:67-80 */
  Obj *o = &e->objs[idx];
  if (o->removed) return;
  e->obj_map[CELL(e, x, y)] = idx;
  e->obj_map[CELL(e, o->x, o->y)] = 0;
  e->touched[chunk_of(e, x, y)] = 1;
  o->x = x; o->y = y;
}
/* engine.py:87-93: (material, object) or (None, None) outside the map. */
static void world_get(const CoEnv *e, int x, int y, int *mat, int *obj) {
  if (!inside(e, x, y)) { *mat = M_NONE; *obj = 0; return; }
  *mat = e->mat[CELL(e, x, y)];
  *obj = e->obj_map[CELL(e, x, y)];
}
static int *health_of(CoEnv *e, int idx) {
  return e->objs[idx].type == T_PLAYER ? &e->inventory[I_HEALTH] : &e->objs[idx].health;
}
static void damage(CoEnv *e, int idx, int amount) { /* objects.py:27-29 setter clamps at 0 */
  int *h = health_of(e, idx);
  *h = *h - amount > 0 ? *h - amount : 0;
}
static int is_free(const CoEnv *e, int x, int y, unsigned walkable) { /* objects.py:44-47 */
  int mat, obj;
  world_get(e, x, y, &mat, &obj);
  return obj == 0 && mat != M_NONE && ((walkable >> mat) & 1u);
}
static int obj_move(CoEnv *e, int idx, int dx, int dy, unsigned walkable) { /* objects.py:36-42 */
  Obj *o = &e->objs[idx];
  int tx = o->x + dx, ty = o->y + dy;
  if (is_free(e, tx, ty, walkable)) { world_move(e, idx, tx, ty); return 1; }
  return 0;
}
static int dist_to_player(const CoEnv *e, const Obj *o) { /* objects.py:49-52 */
  return abs(e->objs[1].x - o->x) + abs(e->objs[1].y - o->y);
}
static int sign(int v) { return (v > 0) - (v < 0); }
static void toward_player(const CoEnv *e, const Obj *o, int long_axis, int *dx, int *dy) {
  int ox = e->objs[1].x - o->x, oy = e->objs[1].y - o->y; /* objects.py:54-62 */
  int ax = abs(ox), ay = abs(oy);
  if (long_axis ? ax > ay : ax <= ay) { *dx = sign(ox); *dy = 0; }
  else { *dx = 0; *dy = sign(oy); }
}

/* ---- player: crafter/objects.py:68-261 ------------------------------------------------------ */
static void player_do_object(CoEnv *e, int idx) { /* objects.py:181-209 */
  int dmg = 1;
  if (e->inventory[I_WOOD_SWORD] && dmg < 2) dmg = 2;
  if (e->inventory[I_STONE_SWORD] && dmg < 3) dmg = 3;
  if (e->inventory[I_IRON_SWORD] && dmg < 5) dmg = 5;
  Obj *o = &e->objs[idx];
  if (o->type == T_PLANT) {
    if (o->grown > 300) { /* ripe objects.py:401-403 */
      o->grown = 0;
      e->inventory[I_FOOD] += 4;
      e->achievements[A_EAT_PLANT] += 1;
    }
  } else if (o->type == T_ZOMBIE) {
    damage(e, idx, dmg);
    if (o->health <= 0) e->achievements[A_DEFEAT_ZOMBIE] += 1;
  } else if (o->type == T_SKELETON) {
    damage(e, idx, dmg);
    if (o->health <= 0) e->achievements[A_DEFEAT_SKELETON] += 1;
  } else if (o->type == T_COW) {
    damage(e, idx, dmg);
    if (o->health <= 0) {
      e->inventory[I_FOOD] += 6;
      e->achievements[A_EAT_COW] += 1;
      e->hunger2 = 0;
    }
  }
}
static void player_do_material(CoEnv *e, int tx, int ty, int mat) { /* objects.py:211-229 */
  if (mat == M_WATER) e->thirst2 = 0;
  const CollectRule *rule = NULL;
  for (unsigned i = 0; i < sizeof(COLLECT) / sizeof(COLLECT[0]); ++i)
    if (COLLECT[i].mat == mat) rule = &COLLECT[i];
  if (!rule) return;
  if (rule->req_item >= 0 && e->inventory[rule->req_item] < 1) return;
  e->mat[CELL(e, tx, ty)] = (uint8_t)rule->leaves;
  if (rng_uniform(&e->rng) <= rule->prob) { /* drawn even when probability is 1 (:226) */
    e->inventory[rule->recv_item] += 1;
    e->achievements[rule->recv_ach] += 1;
  }
}
static void player_place(CoEnv *e, int which, int tx, int ty, int mat) { /* objects.py:231-247 */
  int m2, obj;
  world_get(e, tx, ty, &m2, &obj);
  if (obj) return;
  const PlaceRule *r = &PLACE[which];
  if (mat == M_NONE || !((r->where >> mat) & 1u)) return;
  if (e->inventory[r->item] < r->amount) return;
  e->inventory[r->item] -= r->amount;
  if (r->result_mat >= 0) {
    e->mat[CELL(e, tx, ty)] = (uint8_t)r->result_mat;
  } else {
    Obj p = {0};
    p.type = T_PLANT; p.x = tx; p.y = ty; p.health = 1; p.grown = 0; /* objects.py:389-392 */
    world_add(e, p);
  }
  e->achievements[r->ach] += 1;
}
static void player_make(CoEnv *e, int which) { /* objects.py:249-261 + engine.py:95-103 */
  const Obj *p = &e->objs[1];
  unsigned nearby = 0;
  /* numpy slice [x-1:x+2, y-1:y+2]: a negative start wraps and yields an empty window (Q7). */
  if (p->x - 1 >= 0 && p->y - 1 >= 0)
    for (int x = p->x - 1; x <= p->x + 1 && x < e->aw; ++x)
      for (int y = p->y - 1; y <= p->y + 1 && y < e->ah; ++y)
        nearby |= MB(e->mat[CELL(e, x, y)]);
  const MakeRule *r = &MAKE[which];
  if (!(nearby & MB(M_TABLE))) return;
  if (r->need_furnace && !(nearby & MB(M_FURNACE))) return;
  if (e->inventory[I_WOOD] < r->wood || e->inventory[I_STONE] < r->stone ||
      e->inventory[I_COAL] < r->coal || e->inventory[I_IRON] < r->iron) return;
  e->inventory[I_WOOD] -= r->wood;
  e->inventory[I_STONE] -= r->stone;
  e->inventory[I_COAL] -= r->coal;
  e->inventory[I_IRON] -= r->iron;
  e->inventory[r->gives] += 1;
  e->achievements[r->ach] += 1;
}
static void player_update(CoEnv *e) { /* objects.py:99-131 */
  Obj *p = &e->objs[1];
  int tx = p->x + DIRS[p->facing][0], ty = p->y + DIRS[p->facing][1];
  int mat, obj;
  world_get(e, tx, ty, &mat, &obj);
  int action = e->action;
  if (e->sleeping) {
    if (e->inventory[I_ENERGY] < 9) action = ACT_SLEEP;
    else { e->sleeping = 0; e->achievements[A_WAKE_UP] += 1; }
  }
  if (action == ACT_NOOP) {
  } else if (action >= ACT_LEFT && action <= ACT_DOWN) { /* objects.py:174-179 */
    p->facing = action - ACT_LEFT;
    obj_move(e, 1, DIRS[p->facing][0], DIRS[p->facing][1], WALKABLE_PLAYER);
    p = &e->objs[1];
    if (e->mat[CELL(e, p->x, p->y)] == M_LAVA) e->inventory[I_HEALTH] = 0;
  } else if (action == ACT_DO && obj) {
    player_do_object(e, obj);
  } else if (action == ACT_DO) {
    player_do_material(e, tx, ty, mat);
  } else if (action == ACT_SLEEP) {
    if (e->inventory[I_ENERGY] < 9) e->sleeping = 1;
  } else if (action >= ACT_PLACE_STONE && action <= ACT_PLACE_PLANT) {
    player_place(e, action - ACT_PLACE_STONE, tx, ty, mat);
  } else if (action >= ACT_MAKE_WOOD_PICKAXE && action <= ACT_MAKE_IRON_SWORD) {
    player_make(e, action - ACT_MAKE_WOOD_PICKAXE);
  }
  /* _update_life_stats objects.py:133-152 (half units: hunger2 = 2*_hunger ...) */
  e->hunger2 += e->sleeping ? 1 : 2;
  if (e->hunger2 > 50) { e->hunger2 = 0; e->inventory[I_FOOD] -= 1; }
  e->thirst2 += e->sleeping ? 1 : 2;
  if (e->thirst2 > 40) { e->thirst2 = 0; e->inventory[I_DRINK] -= 1; }
  if (e->sleeping) e->fatigue = e->fatigue - 1 < 0 ? e->fatigue - 1 : 0;
  else e->fatigue += 1;
  if (e->fatigue < -10) { e->fatigue = 0; e->inventory[I_ENERGY] += 1; }
  if (e->fatigue > 30) { e->fatigue = 0; e->inventory[I_ENERGY] -= 1; }
  /* _degen_or_regen_health objects.py:154-167 */
  int ok = e->inventory[I_FOOD] > 0 && e->inventory[I_DRINK] > 0 &&
           (e->inventory[I_ENERGY] > 0 || e->sleeping);
  if (ok) e->recover2 += e->sleeping ? 4 : 2;
  else e->recover2 -= e->sleeping ? 1 : 2;
  if (e->recover2 > 50) { e->recover2 = 0; e->inventory[I_HEALTH] += 1; }
  if (e->recover2 < -30) {
    e->recover2 = 0;
    e->inventory[I_HEALTH] = e->inventory[I_HEALTH] - 1 > 0 ? e->inventory[I_HEALTH] - 1 : 0;
  }
  for (int i = 0; i < N_ITEMS; ++i) { /* objects.py:126-128 */
    if (e->inventory[i] > 9) e->inventory[i] = 9;
    if (e->inventory[i] < 0) e->inventory[i] = 0;
  }
  /* _wake_up_when_hurt objects.py:169-172 */
  if (e->inventory[I_HEALTH] < e->p_last_health) e->sleeping = 0;
  e->p_last_health = e->inventory[I_HEALTH];
}

/* ---- creatures: crafter/objects.py:264-411 -------------------------------------------------- */
static void random_dir(CoEnv *e, int *dx, int *dy) { /* objects.py:64-65 */
  uint32_t i = rng_randint(&e->rng, 4);
  *dx = DIRS[i][0]; *dy = DIRS[i][1];
}
static void cow_update(CoEnv *e, int idx) { /* objects.py:274-279 */
  if (e->objs[idx].health <= 0) world_remove(e, idx);
  if (rng_uniform(&e->rng) < 0.5) {
    int dx, dy;
    random_dir(e, &dx, &dy);
    obj_move(e, idx, dx, dy, WALKABLE);
  }
}
static void zombie_update(CoEnv *e, int idx) { /* objects.py:294-312 */
  Obj *o = &e->objs[idx];
  if (o->health <= 0) world_remove(e, idx);
  int dist = dist_to_player(e, o), dx, dy;
  if (dist <= 8 && rng_uniform(&e->rng) < 0.9) {
    int long_axis = rng_uniform(&e->rng) < 0.8;
    toward_player(e, o, long_axis, &dx, &dy);
    obj_move(e, idx, dx, dy, WALKABLE);
  } else {
    random_dir(e, &dx, &dy);
    obj_move(e, idx, dx, dy, WALKABLE);
  }
  o = &e->objs[idx];
  dist = dist_to_player(e, o);
  if (dist <= 1) {
    if (o->cooldown) {
      o->cooldown -= 1;
    } else {
      damage(e, 1, e->sleeping ? 7 : 2);
      o->cooldown = 5;
    }
  }
}
static void skeleton_update(CoEnv *e, int idx) { /* objects.py:327-351 */
  Obj *o = &e->objs[idx];
  int dx, dy;
  if (o->health <= 0) world_remove(e, idx);
  o->reload = o->reload - 1 > 0 ? o->reload - 1 : 0;
  int dist = dist_to_player(e, o);
  if (dist <= 3) {
    int long_axis = rng_uniform(&e->rng) < 0.6;
    toward_player(e, o, long_axis, &dx, &dy);
    if (obj_move(e, idx, -dx, -dy, WALKABLE)) return;
    o = &e->objs[idx];
  }
  if (dist <= 5 && rng_uniform(&e->rng) < 0.5) {
    toward_player(e, o, 1, &dx, &dy); /* _shoot objects.py:343-351 */
    if (o->reload > 0) return;
    if (dx == 0 && dy == 0) return;
    int px = o->x + dx, py = o->y + dy;
    if (is_free(e, px, py, WALKABLE_ARROW)) {
      Obj a = {0};
      a.type = T_ARROW; a.x = px; a.y = py; a.health = 0;
      a.facing = dx < 0 ? 0 : dx > 0 ? 1 : dy < 0 ? 2 : 3;
      world_add(e, a);
      e->objs[idx].reload = 4;
    }
  } else if (dist <= 8 && rng_uniform(&e->rng) < 0.3) {
    int long_axis = rng_uniform(&e->rng) < 0.6;
    toward_player(e, o, long_axis, &dx, &dy);
    obj_move(e, idx, dx, dy, WALKABLE);
  } else if (rng_uniform(&e->rng) < 0.2) {
    random_dir(e, &dx, &dy);
    obj_move(e, idx, dx, dy, WALKABLE);
  }
}
static void arrow_update(CoEnv *e, int idx) { /* objects.py:373-384 */
  Obj *o = &e->objs[idx];
  int dx = DIRS[o->facing][0], dy = DIRS[o->facing][1];
  int tx = o->x + dx, ty = o->y + dy, mat, obj;
  world_get(e, tx, ty, &mat, &obj);
  if (obj) {
    damage(e, obj, 2);
    world_remove(e, idx);
  } else if (mat == M_NONE || !((WALKABLE_ARROW >> mat) & 1u)) {
    world_remove(e, idx);
    if (mat == M_TABLE || mat == M_FURNACE) e->mat[CELL(e, tx, ty)] = M_PATH;
  } else {
    obj_move(e, idx, dx, dy, WALKABLE_ARROW);
  }
}
static void plant_update(CoEnv *e, int idx) { /* objects.py:405-411 */
  Obj *o = &e->objs[idx];
  o->grown += 1;
  int hurt = 0;
  for (int d = 0; d < 4; ++d) {
    int mat, obj;
    world_get(e, o->x + DIRS[d][0], o->y + DIRS[d][1], &mat, &obj);
    if (obj) {
      int t = e->objs[obj].type;
      if (t == T_ZOMBIE || t == T_SKELETON || t == T_COW) hurt = 1;
    }
  }
  if (hurt) damage(e, idx, 1);
  if (o->health <= 0) world_remove(e, idx);
}

/* ---- worldgen: crafter/worldgen.py ---------------------------------------------------------- */
static double n3(const CoEnv *e, double x, double y, double z, double size) {
  return osn_noise3(e->perm, e->pgi, x / size, y / size, z); /* worldgen.py:79-91, one octave */
}
static void set_material(CoEnv *e, int x, int y) { /* worldgen.py:21-61 */
  const Obj *p = &e->objs[1];
  rng_ctx(&e->rng, D_WG_MAT, (uint32_t)CELL(e, x, y), 0, 0);
  double fx = x, fy = y;
  int ddx = x - p->x, ddy = y - p->y;
  double start = 4 - sqrt((double)(ddx * ddx + ddy * ddy));
  start += 2 * n3(e, fx, fy, 8, 3);
  start = 1 / (1 + exp(-start));
  /* _simplex(x, y, 3, {15: 1, 5: 0.15}, False): value = 0 + 1*n + 0.15*n, unnormalised */
  double water = (0 + 1 * n3(e, fx, fy, 3, 15)) + 0.15 * n3(e, fx, fy, 3, 5);
  water = water + 0.1;
  water -= 2 * start;
  double mountain = (0 + 1 * n3(e, fx, fy, 0, 15)) + 0.3 * n3(e, fx, fy, 0, 5);
  mountain /= (1 + 0.3);
  mountain -= 4 * start + 0.3 * water;
  int m;
  if (start > 0.5) {
    m = M_GRASS;
  } else if (mountain > 0.15) {
    if (n3(e, fx, fy, 6, 7) > 0.15 && mountain > 0.3) m = M_PATH; /* cave */
    else if (n3(e, 2 * x, fy / 5, 7, 3) > 0.4) { m = M_PATH; e->tunnels[CELL(e, x, y)] = 1; }
    else if (n3(e, fx / 5, 2 * y, 7, 3) > 0.4) { m = M_PATH; e->tunnels[CELL(e, x, y)] = 1; }
    else if (n3(e, fx, fy, 1, 8) > 0 && rng_uniform(&e->rng) > 0.85) m = M_COAL;
    else if (n3(e, fx, fy, 2, 6) > 0.4 && rng_uniform(&e->rng) > 0.75) m = M_IRON;
    else if (mountain > 0.18 && rng_uniform(&e->rng) > 0.994) m = M_DIAMOND;
    else if (mountain > 0.3 && n3(e, fx, fy, 6, 5) > 0.35) m = M_LAVA;
    else m = M_STONE;
  } else if (0.25 < water && water <= 0.35 && n3(e, fx, fy, 4, 9) > -0.2) {
    m = M_SAND;
  } else if (0.3 < water) {
    m = M_WATER;
  } else {
    if (n3(e, fx, fy, 5, 7) > 0 && rng_uniform(&e->rng) > 0.8) m = M_TREE;
    else m = M_GRASS;
  }
  e->mat[CELL(e, x, y)] = (uint8_t)m;
}
static void set_object(CoEnv *e, int x, int y) { /* worldgen.py:64-76 */
  const Obj *p = &e->objs[1];
  rng_ctx(&e->rng, D_WG_OBJ, (uint32_t)CELL(e, x, y), 0, 0);
  int ddx = x - p->x, ddy = y - p->y;
  double dist = sqrt((double)(ddx * ddx + ddy * ddy));
  int m = e->mat[CELL(e, x, y)];
  Obj o = {0};
  o.x = x; o.y = y;
  if (!((WALKABLE >> m) & 1u)) {
  } else if (dist > 3 && m == M_GRASS && rng_uniform(&e->rng) > 0.985) {
    o.type = T_COW; o.health = 3; world_add(e, o); /* objects.py:266-268 */
  } else if (dist > 10 && rng_uniform(&e->rng) > 0.993) {
    o.type = T_ZOMBIE; o.health = 5; world_add(e, o); /* objects.py:284-288 */
  } else if (m == M_PATH && e->tunnels[CELL(e, x, y)] && rng_uniform(&e->rng) > 0.95) {
    o.type = T_SKELETON; o.health = 3; world_add(e, o); /* objects.py:317-321 */
  }
}

/* ---- env: crafter/env.py -------------------------------------------------------------------- */
static void update_time(CoEnv *e) { /* env.py:135-139 via the host table */
  int i = e->step < e->n_daylight ? e->step : e->n_daylight - 1;
  e->daylight = e->daylight_table[i];
}

void co_reset(CoEnv *e) { /* env.py:70-81 */
  int cells = e->aw * e->ah;
  e->episode += 1;
  e->step = 0;
  memset(&e->rng, 0, sizeof(e->rng)); /* engine.py:33-39 */
  e->rng.seed = (uint32_t)co_world_seed(e->seed, e->episode);
  memset(e->mat, 0, cells);
  memset(e->obj_map, 0, sizeof(int32_t) * cells);
  memset(e->tunnels, 0, cells);
  memset(e->touched, 0, e->ncx * e->ncy);
  e->n_slots = 1;
  update_time(e);
  Obj p = {0}; /* objects.py:70-82 */
  p.type = T_PLAYER; p.x = e->aw / 2; p.y = e->ah / 2; p.facing = 3;
  static const int initial[N_ITEMS] = {9, 9, 9, 9}; /* data.yaml:39-55 */
  memcpy(e->inventory, initial, sizeof(initial));
  memset(e->achievements, 0, sizeof(e->achievements));
  e->action = ACT_NOOP; e->sleeping = 0;
  e->p_last_health = 9; e->hunger2 = e->thirst2 = e->fatigue = e->recover2 = 0;
  e->last_health = 9;
  world_add(e, p);
  e->unlocked = 0;
  /* worldgen.py:10-18 */
  rng_ctx(&e->rng, D_SEED, 0, 0, 0);
  osn_init((int64_t)rng_randint(&e->rng, 2147483647u), e->perm, e->pgi);
  for (int x = 0; x < e->aw; ++x)
    for (int y = 0; y < e->ah; ++y) set_material(e, x, y);
  for (int x = 0; x < e->aw; ++x)
    for (int y = 0; y < e->ah; ++y) set_object(e, x, y);
}

static void balance_object(CoEnv *e, int cx, int cy, int cls_idx, int type, int material,
                           int span_dist, int despan_dist, double spawn_prob,
                           double despawn_prob, const int *snapshot, int n_snapshot) {
  /* env.py:157-179 */
  int xmin = cx * 12, ymin = cy * 12;
  int xmax = xmin + 12 < e->aw ? xmin + 12 : e->aw;
  int ymax = ymin + 12 < e->ah ? ymin + 12 : e->ah;
  rng_ctx(&e->rng, D_BALANCE, (uint32_t)e->step, (uint32_t)(cx * e->ncy + cy), (uint32_t)cls_idx);
  int n = 0, space = 0;
  for (int i = 0; i < n_snapshot; ++i) {
    const Obj *o = &e->objs[snapshot[i]];
    if (!o->removed && o->type == type && o->x / 12 == cx && o->y / 12 == cy) n++;
  }
  for (int x = xmin; x < xmax; ++x)
    for (int y = ymin; y < ymax; ++y) space += e->mat[CELL(e, x, y)] == material;
  double light = e->daylight, tmin, tmax; /* env.py:143-155 */
  if (type == T_ZOMBIE) { tmin = space < 50 ? 0 : 3.5 - 3 * light; tmax = 3.5 - 3 * light; }
  else if (type == T_SKELETON) { tmin = space < 6 ? 0 : 1; tmax = 2; }
  else { tmin = space < 30 ? 0 : 1; tmax = 1.5 + light; }
  if (n < (int)tmin && rng_uniform(&e->rng) < spawn_prob) {
    int pick = (int)rng_randint(&e->rng, (uint32_t)space), k = 0, px = -1, py = -1;
    for (int x = xmin; x < xmax && px < 0; ++x)
      for (int y = ymin; y < ymax; ++y)
        if (e->mat[CELL(e, x, y)] == material && k++ == pick) { px = x; py = y; break; }
    int empty = e->obj_map[CELL(e, px, py)] == 0;
    int away = abs(e->objs[1].x - px) + abs(e->objs[1].y - py) >= span_dist;
    if (empty && away) {
      Obj o = {0};
      o.type = type; o.x = px; o.y = py;
      o.health = type == T_ZOMBIE ? 5 : 3;
      world_add(e, o);
    }
  } else if (n > (int)tmax && rng_uniform(&e->rng) < despawn_prob) {
    int pick = (int)rng_randint(&e->rng, (uint32_t)n), k = 0;
    for (int i = 0; i < n_snapshot; ++i) {
      const Obj *o = &e->objs[snapshot[i]];
      if (!o->removed && o->type == type && o->x / 12 == cx && o->y / 12 == cy && k++ == pick) {
        if (dist_to_player(e, o) >= despan_dist) world_remove(e, snapshot[i]);
        break;
      }
    }
  }
}

void co_render(CoEnv *e, uint8_t *obs);

void co_step(CoEnv *e, int action, double *reward, int *done) { /* env.py:83-118 */
  e->step += 1;
  update_time(e);
  e->action = action;
  rng_ctx(&e->rng, D_UPDATE, (uint32_t)e->step, 0, 0);
  int n0 = e->n_slots; /* snapshot engine.py:41-44 */
  int radius = 2 * (e->vw > e->vh ? e->vw : e->vh);
  for (int i = 1; i < n0; ++i) {
    Obj *o = &e->objs[i];
    if (o->removed) continue;
    if (dist_to_player(e, o) >= radius) continue;
    switch (o->type) {
      case T_PLAYER: player_update(e); break;
      case T_COW: cow_update(e, i); break;
      case T_ZOMBIE: zombie_update(e, i); break;
      case T_SKELETON: skeleton_update(e, i); break;
      case T_ARROW: arrow_update(e, i); break;
      case T_PLANT: plant_update(e, i); break;
    }
  }
  if (e->step % 10 == 0) { /* env.py:90-95, chunks in sorted key order, members in slot order */
    int n_snapshot = 0;
    int *snapshot = (int *)malloc(sizeof(int) * e->n_slots);
    for (int i = 1; i < e->n_slots; ++i)
      if (!e->objs[i].removed) snapshot[n_snapshot++] = i;
    uint8_t *touched0 = (uint8_t *)malloc(e->ncx * e->ncy);
    memcpy(touched0, e->touched, e->ncx * e->ncy);
    for (int cx = 0; cx < e->ncx; ++cx)
      for (int cy = 0; cy < e->ncy; ++cy) {
        if (!touched0[cx * e->ncy + cy]) continue;
        balance_object(e, cx, cy, 0, T_ZOMBIE, M_GRASS, 6, 0, 0.3, 0.4, snapshot, n_snapshot);
        balance_object(e, cx, cy, 1, T_SKELETON, M_PATH, 7, 7, 0.1, 0.1, snapshot, n_snapshot);
        balance_object(e, cx, cy, 2, T_COW, M_GRASS, 5, 5, 0.01, 0.1, snapshot, n_snapshot);
      }
    free(snapshot);
    free(touched0);
  }
  int health = e->inventory[I_HEALTH]; /* env.py:97-107 */
  double r = (double)(health - e->last_health) / 10;
  e->last_health = health;
  uint32_t now = 0;
  for (int i = 0; i < N_ACH; ++i)
    if (e->achievements[i] > 0) now |= 1u << i;
  if (now & ~e->unlocked) { e->unlocked |= now; r += 1.0; }
  int dead = health <= 0;
  int over = e->length && e->step >= e->length;
  *done = dead || over;
  *reward = e->reward_flag ? r : 0.0;
}

/* ---- render: crafter/engine.py:155-248,267-284, crafter/env.py:120-130 ---------------------- */
static void draw_alpha(uint8_t *canvas, int ch, int x0, int y0, const uint8_t *tex, int w, int h) {
  /* engine.py:276-284; canvas[x][y][3] with height ch; tex[x][y][4] */
  for (int x = 0; x < w; ++x)
    for (int y = 0; y < h; ++y) {
      const uint8_t *t = tex + (x * h + y) * 4;
      uint8_t *c = canvas + ((x0 + x) * ch + (y0 + y)) * 3;
      float alpha = (float)t[3] / 255.0f;
      for (int k = 0; k < 3; ++k) {
        float tv = (float)t[k] / 255.0f, cv = (float)c[k] / 255.0f;
        float blended = alpha * tv + (1.0f - alpha) * cv;
        c[k] = (uint8_t)(255.0f * blended);
      }
    }
}
static int luma(const uint8_t *p) { /* PIL convert('L') */
  return (p[0] * 19595 + p[1] * 38470 + p[2] * 7471 + 0x8000) >> 16;
}
static int obj_texture(const CoEnv *e, const Obj *o) {
  switch (o->type) { /* objects.py:84-93,270,290,323,360-367,394-399 */
    case T_PLAYER: return e->sleeping ? 4 : o->facing;
    case T_COW: return 5;
    case T_ZOMBIE: return 6;
    case T_SKELETON: return 7;
    case T_ARROW: return 8 + o->facing;
    default: return o->grown > 300 ? 13 : 12;
  }
}

void co_render(CoEnv *e, uint8_t *obs) {
  const Tex *t = &e->tex;
  int lw = e->gx * t->ux, lh = e->gy * t->uy;        /* local view canvas */
  int iw_ = e->vw * t->ux, ih_ = e->item_rows * t->uy; /* item view canvas */
  uint8_t *local = (uint8_t *)malloc(lw * lh * 3);
  uint8_t *items = (uint8_t *)calloc(iw_ * ih_ * 3, 1);
  double *out = (double *)malloc(sizeof(double) * lw * lh * 3);
  memset(local, 127, lw * lh * 3); /* engine.py:168 */
  const Obj *p = &e->objs[1];
  int offx = e->gx / 2, offy = e->gy / 2; /* engine.py:161 */
  for (int i = 0; i < e->gx; ++i)
    for (int j = 0; j < e->gy; ++j) { /* engine.py:169-175 */
      int wx = p->x + i - offx, wy = p->y + j - offy;
      if (!inside(e, wx, wy)) continue;
      const uint8_t *tex = t->mat_tex + e->mat[CELL(e, wx, wy)] * t->ux * t->uy * 3;
      for (int x = 0; x < t->ux; ++x)
        memcpy(local + ((i * t->ux + x) * lh + j * t->uy) * 3, tex + x * t->uy * 3, t->uy * 3);
    }
  for (int s = 1; s < e->n_slots; ++s) { /* engine.py:176-181 */
    const Obj *o = &e->objs[s];
    if (o->removed) continue;
    int i = o->x - p->x + offx, j = o->y - p->y + offy;
    if (i < 0 || i >= e->gx || j < 0 || j >= e->gy) continue;
    draw_alpha(local, lh, i * t->ux, j * t->uy,
               t->obj_tex + obj_texture(e, o) * t->ux * t->uy * 4, t->ux, t->uy);
  }
  /* _light engine.py:189-196 */
  double daylight = e->daylight;
  uint32_t w4[4] = {0, 0, 0, 0};
  for (int x = 0; x < lw; ++x)
    for (int y = 0; y < lh; ++y) {
      const uint8_t *c = local + (x * lh + y) * 3;
      uint8_t night[3] = {c[0], c[1], c[2]};
      if (daylight < 0.5) { /* _noise engine.py:208-211 */
        philox(e->rng.seed, D_NOISE, (uint32_t)x >> 2, (uint32_t)e->step, (uint32_t)y, 0, w4);
        double u = 32.0 + (127.0 - 32.0) * ((double)w4[x & 3] * (1.0 / 4294967296.0));
        double mask = (2 * (0.5 - daylight)) * t->vignette[x * lh + y];
        for (int k = 0; k < 3; ++k)
          night[k] = (uint8_t)((1 - mask) * (double)c[k] + mask * u);
      }
      int L = luma(night); /* ImageEnhance.Color(...).enhance(0.4) == blend(grey, image, 0.4) */
      for (int k = 0; k < 3; ++k) {
        uint8_t enh = (uint8_t)((float)L + 0.4f * (float)((int)night[k] - L));
        static const double tint[3] = {0, 16, 64};
        double n = (1 - 0.5) * (double)enh + 0.5 * tint[k]; /* _tint engine.py:204-206 */
        out[(x * lh + y) * 3 + k] = daylight * (double)c[k] + (1 - daylight) * n;
      }
      if (e->sleeping) { /* _sleep engine.py:198-202 */
        uint8_t q[3] = {(uint8_t)out[(x * lh + y) * 3], (uint8_t)out[(x * lh + y) * 3 + 1],
                        (uint8_t)out[(x * lh + y) * 3 + 2]};
        int G = luma(q);
        static const double tint2[3] = {0, 0, 16};
        for (int k = 0; k < 3; ++k)
          out[(x * lh + y) * 3 + k] = (1 - 0.5) * (double)G + 0.5 * tint2[k];
      }
    }
  /* ItemView engine.py:227-248 */
  for (int idx = 0; idx < N_ITEMS; ++idx) {
    int amount = e->inventory[idx];
    if (amount < 1) continue;
    draw_alpha(items, ih_, t->item_pos[idx][0], t->item_pos[idx][1],
               t->item_tex + idx * t->iw * t->ih * 4, t->iw, t->ih);
    int d = amount <= 9 ? amount : 0; /* slot 0 holds 'unknown' */
    draw_alpha(items, ih_, t->digit_pos[idx][0], t->digit_pos[idx][1],
               t->digit_tex + d * t->dw * t->dh * 4, t->dw, t->dh);
  }
  /* env.py:120-130: concat on axis 1, paste at border, transpose to (H, W, 3) */
  int bx = (e->sw - t->ux * e->vw) / 2, by = (e->sh - t->uy * e->vh) / 2;
  memset(obs, 0, (size_t)e->sw * e->sh * 3);
  for (int x = 0; x < lw; ++x) {
    for (int y = 0; y < lh; ++y)
      for (int k = 0; k < 3; ++k)
        obs[((by + y) * e->sw + (bx + x)) * 3 + k] = (uint8_t)out[(x * lh + y) * 3 + k];
    for (int y = 0; y < ih_; ++y)
      for (int k = 0; k < 3; ++k)
        obs[((by + lh + y) * e->sw + (bx + x)) * 3 + k] = items[(x * ih_ + y) * 3 + k];
  }
  free(local); free(items); free(out);
}

/* ---- C interface for ctypes ----------------------------------------------------------------- */
CoEnv *co_create(int aw, int ah, int vw, int vh, int sw, int sh, int length, int reward_flag,
                 int64_t seed) {
  CoEnv *e = (CoEnv *)calloc(1, sizeof(CoEnv));
  e->aw = aw; e->ah = ah; e->vw = vw; e->vh = vh; e->sw = sw; e->sh = sh;
  e->length = length; e->reward_flag = reward_flag; e->seed = seed;
  e->item_rows = (N_ITEMS + vw - 1) / vw; /* env.py:42 */
  e->gx = vw; e->gy = vh - e->item_rows;
  e->ncx = (aw + 11) / 12; e->ncy = (ah + 11) / 12;
  e->mat = (uint8_t *)calloc(aw * ah, 1);
  e->obj_map = (int32_t *)calloc(aw * ah, sizeof(int32_t));
  e->tunnels = (uint8_t *)calloc(aw * ah, 1);
  e->touched = (uint8_t *)calloc(e->ncx * e->ncy, 1);
  e->cap_slots = 64;
  e->objs = (Obj *)calloc(e->cap_slots, sizeof(Obj));
  e->n_slots = 1;
  return e;
}
void co_destroy(CoEnv *e) {
  free(e->mat); free(e->obj_map); free(e->tunnels); free(e->touched); free(e->objs);
  free(e->tex.mat_tex); free(e->tex.obj_tex); free(e->tex.item_tex); free(e->tex.digit_tex);
  free(e->tex.vignette); free((void *)e->daylight_table);
  free(e);
}
static void *dup(const void *src, size_t n) { void *p = malloc(n); memcpy(p, src, n); return p; }
void co_set_tables(CoEnv *e, int ux, int uy, int iw, int ih, int dw, int dh, const int *item_pos,
                   const int *digit_pos, const uint8_t *mat_tex, const uint8_t *obj_tex,
                   const uint8_t *item_tex, const uint8_t *digit_tex, const double *vignette,
                   const double *daylight_table, int n_daylight) {
  Tex *t = &e->tex;
  t->ux = ux; t->uy = uy; t->iw = iw; t->ih = ih; t->dw = dw; t->dh = dh;
  memcpy(t->item_pos, item_pos, sizeof(t->item_pos));
  memcpy(t->digit_pos, digit_pos, sizeof(t->digit_pos));
  t->mat_tex = (uint8_t *)dup(mat_tex, 13 * ux * uy * 3);
  t->obj_tex = (uint8_t *)dup(obj_tex, 14 * ux * uy * 4);
  t->item_tex = (uint8_t *)dup(item_tex, 16 * iw * ih * 4);
  t->digit_tex = (uint8_t *)dup(digit_tex, 10 * dw * dh * 4);
  t->vignette = (double *)dup(vignette, sizeof(double) * e->gx * ux * e->gy * uy);
  e->daylight_table = (const double *)dup(daylight_table, sizeof(double) * n_daylight);
  e->n_daylight = n_daylight;
}
void co_set_episode(CoEnv *e, int64_t episode) { e->episode = episode; }
void co_set_inventory(CoEnv *e, int item, int value) {
  e->inventory[item] = value;
  if (item == I_HEALTH) { e->last_health = value; e->p_last_health = value; }
}
int co_num_objects(const CoEnv *e) {
  int n = 0;
  for (int i = 1; i < e->n_slots; ++i) n += !e->objs[i].removed;
  return n;
}
void co_export_objects(const CoEnv *e, int32_t *rows) { /* layout: oracle/canon.py */
  for (int i = 1; i < e->n_slots; ++i) {
    const Obj *o = &e->objs[i];
    if (o->removed) continue;
    int a = 0, b = 0;
    switch (o->type) {
      case T_PLAYER: a = o->facing; b = e->sleeping; break;
      case T_ZOMBIE: a = o->cooldown; break;
      case T_SKELETON: a = o->reload; break;
      case T_ARROW: a = o->facing; break;
      case T_PLANT: a = o->grown; break;
    }
    rows[0] = o->type; rows[1] = o->x; rows[2] = o->y;
    rows[3] = o->type == T_PLAYER ? e->inventory[I_HEALTH] : o->health;
    rows[4] = a; rows[5] = b;
    rows += 6;
  }
}
void co_export_mat(const CoEnv *e, uint8_t *out) { memcpy(out, e->mat, e->aw * e->ah); }
void co_export_player(const CoEnv *e, int64_t *v) {
  int k = 0;
  for (int i = 0; i < N_ITEMS; ++i) v[k++] = e->inventory[i];
  for (int i = 0; i < N_ACH; ++i) v[k++] = e->achievements[i];
  v[k++] = e->hunger2; v[k++] = e->thirst2; v[k++] = e->fatigue; v[k++] = e->recover2;
  v[k++] = e->sleeping; v[k++] = e->objs[1].facing; v[k++] = e->p_last_health;
  v[k++] = e->objs[1].x; v[k++] = e->objs[1].y; v[k++] = e->last_health; v[k++] = e->unlocked;
}
int co_export_touched(const CoEnv *e, int32_t *out) {
  int n = 0;
  for (int c = 0; c < e->ncx * e->ncy; ++c)
    if (e->touched[c]) out[n++] = c;
  return n;
}
/* Load a canonical state (oracle/canon.py layout, as co_export_* write it) plus the three scalars
 * it does not carry: tests/test_scenarios_golden.py replays reference-recorded corner cases. */
void co_import_state(CoEnv *e, const uint8_t *mat, const int32_t *rows, int n_rows,
                     const int64_t *v, const int32_t *touched, int n_touched, int step,
                     int64_t episode, int64_t world_seed) {
  int cells = e->aw * e->ah;
  memcpy(e->mat, mat, cells);
  memset(e->obj_map, 0, sizeof(int32_t) * cells);
  memset(e->touched, 0, e->ncx * e->ncy);
  e->n_slots = 1;
  for (int i = 0; i < n_rows; ++i, rows += 6) {
    Obj o = {0};
    o.type = rows[0]; o.x = rows[1]; o.y = rows[2]; o.health = rows[3];
    switch (o.type) {
      case T_PLAYER: o.facing = rows[4]; break;
      case T_ZOMBIE: o.cooldown = rows[4]; break;
      case T_SKELETON: o.reload = rows[4]; break;
      case T_ARROW: o.facing = rows[4]; break;
      case T_PLANT: o.grown = rows[4]; break;
    }
    world_add(e, o);
  }
  memset(e->touched, 0, e->ncx * e->ncy); /* exactly the recorded set, not what world_add marked */
  for (int i = 0; i < n_touched; ++i) e->touched[touched[i]] = 1;
  int k = 0;
  for (int i = 0; i < N_ITEMS; ++i) e->inventory[i] = (int)v[k++];
  for (int i = 0; i < N_ACH; ++i) e->achievements[i] = (int)v[k++];
  e->hunger2 = (int)v[k++]; e->thirst2 = (int)v[k++]; e->fatigue = (int)v[k++]; e->recover2 = (int)v[k++];
  e->sleeping = (int)v[k++]; k++; /* facing: on the player's row */ e->p_last_health = (int)v[k++];
  k += 2; /* position: on the player's row */ e->last_health = (int)v[k++]; e->unlocked = (uint32_t)v[k++];
  e->step = step;
  e->episode = episode;
  memset(&e->rng, 0, sizeof(e->rng));
  e->rng.seed = (uint32_t)world_seed;
  update_time(e);
}
double co_daylight(const CoEnv *e) { return e->daylight; }
int co_step_count(const CoEnv *e) { return e->step; }
long co_rng_draws(const CoEnv *e) { return e->rng.draws; }
void co_semantic(const CoEnv *e, uint8_t *out) { /* engine.py:260-264 */
  memcpy(out, e->mat, e->aw * e->ah);
  for (int i = 1; i < e->n_slots; ++i)
    if (!e->objs[i].removed) out[CELL(e, e->objs[i].x, e->objs[i].y)] = 12 + e->objs[i].type;
}

/* Random-policy rollout with reset-on-done, as crafter/run_random.py:36-43; the action stream is a
 * Philox sequence private to the benchmark.  Returns the number of episodes finished. */
int co_run_random(CoEnv *e, int steps, uint32_t policy_seed, int render, uint8_t *obs_buf) {
  int episodes = 0;
  for (int i = 0; i < steps; ++i) {
    uint32_t w[4];
    philox(policy_seed, 0x706f6c69u, (uint32_t)i, 0, 0, 0, w);
    double r; int d;
    co_step(e, (int)(((uint64_t)w[0] * 17) >> 32), &r, &d);
    if (render) co_render(e, obs_buf);
    if (d) { co_reset(e); if (render) co_render(e, obs_buf); episodes++; }
  }
  return episodes;
}

/* Batched convenience for the CPU baseline: one tick (+ render, + reset-on-done) of n envs.
 * Python worker threads call this on disjoint chunks; ctypes drops the GIL. */
void co_step_many(CoEnv **envs, int n, const int32_t *actions, double *rewards, int32_t *dones,
                  uint8_t *obs, int auto_reset) {
  for (int i = 0; i < n; ++i) {
    CoEnv *e = envs[i];
    co_step(e, actions[i], &rewards[i], &dones[i]);
    if (dones[i] && auto_reset) co_reset(e);
    if (obs) co_render(e, obs + (size_t)i * e->sw * e->sh * 3);
  }
}
void co_reset_many(CoEnv **envs, int n, uint8_t *obs) {
  for (int i = 0; i < n; ++i) {
    co_reset(envs[i]);
    if (obs) co_render(envs[i], obs + (size_t)i * envs[i]->sw * envs[i]->sh * 3);
  }
}
/* Row i of the output belongs to envs[i]: frames, semantic maps, player vectors (co_export_player). */
void co_render_many(CoEnv **envs, int n, uint8_t *obs) {
  for (int i = 0; i < n; ++i) co_render(envs[i], obs + (size_t)i * envs[i]->sw * envs[i]->sh * 3);
}
void co_semantic_many(CoEnv **envs, int n, uint8_t *out) {
  for (int i = 0; i < n; ++i) co_semantic(envs[i], out + (size_t)i * envs[i]->aw * envs[i]->ah);
}
void co_export_player_many(CoEnv **envs, int n, int64_t *out) {
  for (int i = 0; i < n; ++i) co_export_player(envs[i], out + (size_t)i * 49);
}
