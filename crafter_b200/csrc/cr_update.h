// One environment tick: Env.step (env.py:83-118) = time -> slot-ordered entity updates ->
// spawn/despawn balance -> reward/done.  One warp owns one environment: the serial, order-dependent
// rules (SURVEY.md F6) run on lane 0 in reference slot order; the warp cooperates on the scans
// (radius filter by ballot, per-chunk creature/material census, slot compaction).
#pragma once
#include "cr_common.h"

namespace cr {

// Per-warp working copy of the player (shared memory on the device).
constexpr int DRAW_TAB = 32;  // one block per lane of the ticking warp
struct PlayerS {
  int32_t inv[N_ITEMS];
  int32_t ach[N_ACH];
  int32_t ps[PS_COUNT];
  uint32_t draw[DRAW_TAB * 2];  // words (w0, w1) of the step's first DRAW_TAB D_UPDATE blocks (draw prefetch)
};

struct EnvRef {
  const Geom *g;
  uint8_t *mat;
  uint16_t *objmap;
  Ent *ents;
  uint32_t *touched;
  PlayerS *P;
  Rng rng;  // D_UPDATE stream of this step (lane 0 only)
  // Shared-memory copies of the first ENT_SMEM slot records (write-through) and of the touched
  // chunk set (written back at the end of the tick).
  Ent *sents;
  uint32_t *stouched;
  int32_t *ccnt;  // [NCH][2] grass / path cells per chunk (incremental census), else null
};

constexpr int ENT_SMEM = 192;  // slots mirrored in shared memory; higher slots go to global memory
CR_DEV Ent rd_ent(const EnvRef &E, int slot) { return slot < ENT_SMEM ? E.sents[slot] : E.ents[slot]; }
CR_DEV void wr_ent(const EnvRef &E, int slot, const Ent &e) {
  if (slot < ENT_SMEM) E.sents[slot] = e;
  E.ents[slot] = e;
}

CR_DEV bool inside(const Geom &g, int x, int y) {  // engine.py:267-268
  return x >= 0 && x < g.W && y >= 0 && y < g.H;
}
CR_DEV int cell_of(const Geom &g, int x, int y) { return x * g.H + y; }
CR_DEV int chunk_of(const Geom &g, int x, int y) { return (x / CHUNK) * g.ncy + (y / CHUNK); }

// Grid accessors.  The serial update runs on one lane and is bound by dependent-load latency, so
// the lanes that found an in-radius object first pull its neighbourhood into L1 (grid_prefetch);
// the later accesses of lane 0 then hit L1 instead of L2.
CR_DEV int rd_mat(const EnvRef &E, int x, int y) { return E.mat[cell_of(*E.g, x, y)]; }
CR_DEV int rd_obj(const EnvRef &E, int x, int y) { return E.objmap[cell_of(*E.g, x, y)]; }
// Every terrain write of the tick goes through here (collect, place, arrows into tables): with the
// incremental census the chunk's grass / path counts follow the write.
CR_DEV void wr_mat(const EnvRef &E, int x, int y, int v) {
  const Geom &g = *E.g;
  uint8_t *p = E.mat + cell_of(g, x, y);
  if (g.incr_census) {
    const int old = *p & 0x0F, c = chunk_of(g, x, y) * 2;
    if (old == M_GRASS) E.ccnt[c] -= 1; else if (old == M_PATH) E.ccnt[c + 1] -= 1;
    if (v == M_GRASS) E.ccnt[c] += 1; else if (v == M_PATH) E.ccnt[c + 1] += 1;
  }
  *p = (uint8_t)v;
}
CR_DEV void wr_obj(const EnvRef &E, int x, int y, int v) { E.objmap[cell_of(*E.g, x, y)] = (uint16_t)v; }
CR_DEV void cr_prefetch(const void *p) {
#if !defined(CR_HOSTSIM) && !defined(CR_SIMT)
  asm volatile("prefetch.global.L1 [%0];" ::"l"(p));
#else
  (void)p;
#endif
}
// The three grid rows around (x, y): every cell an object at (x, y) can read this tick.
CR_DEV void grid_prefetch(const EnvRef &E, int x, int y) {
  const Geom &g = *E.g;
  for (int dx = -1; dx <= 1; ++dx) {
    const int xx = x + dx;
    if (xx < 0 || xx >= g.W) continue;
    const int c = xx * g.H + imax(0, y - 1);
    cr_prefetch(E.mat + c);
    cr_prefetch(E.objmap + c);
    const int c2 = imin(c + 2, g.NC - 1);  // a 3-cell span can straddle a 128-byte line
    cr_prefetch(E.mat + c2);
    cr_prefetch(E.objmap + c2);
  }
}

// engine.py:87-93: (material, object) of a cell, (None, None) outside the map.
CR_DEV void w_get(const EnvRef &E, int x, int y, int &mat, int &slot) {
  if (!inside(*E.g, x, y)) { mat = M_NONE; slot = 0; return; }
  mat = rd_mat(E, x, y);
  slot = rd_obj(E, x, y);
}
CR_DEV void w_touch(const EnvRef &E, int x, int y) {  // defaultdict key creation, engine.py:57,79
  int c = chunk_of(*E.g, x, y);
  E.stouched[c >> 5] |= 1u << (c & 31);
}
// engine.py:50-57.  Slots are append-only between compactions; returns 0 when the arena is full.
CR_DEV int w_add(EnvRef &E, const Ent &rec) {
  int n = E.P->ps[PS_NSLOTS];
  if (n >= E.g->CAP) { E.P->ps[PS_ERROR] |= ERR_SLOT_OVERFLOW; return 0; }
  E.P->ps[PS_NSLOTS] = n + 1;
  wr_ent(E, n, rec);
  wr_obj(E, rec.x, rec.y, n);
  w_touch(E, rec.x, rec.y);
  return n;
}
// engine.py:67-80 for a live object.
CR_DEV void w_move(EnvRef &E, int slot, Ent &rec, int nx, int ny) {
  wr_obj(E, nx, ny, slot);
  wr_obj(E, rec.x, rec.y, 0);
  w_touch(E, nx, ny);
  rec.x = (int16_t)nx; rec.y = (int16_t)ny;
}
CR_DEV bool is_free(const EnvRef &E, int x, int y, unsigned walkable) {  // objects.py:44-47
  int mat, slot;
  w_get(E, x, y, mat, slot);
  return slot == 0 && mat != M_NONE && ((walkable >> mat) & 1u);
}
// objects.py:36-42.  A removed object still evaluates is_free and reports success, but
// World.move ignores it (engine.py:68) -- the "ghost" update of a dying mob (SURVEY.md Q3).
CR_DEV bool obj_move(EnvRef &E, int slot, Ent &rec, bool removed, int dx, int dy, unsigned walkable) {
  int tx = rec.x + dx, ty = rec.y + dy;
  if (!is_free(E, tx, ty, walkable)) return false;
  if (!removed) w_move(E, slot, rec, tx, ty);
  return true;
}
// Object.health setter clamps at zero (objects.py:27-29); slot 1 is the player.
CR_DEV void damage_slot(EnvRef &E, int slot, int amount) {
  if (slot == 1) {
    E.P->inv[I_HEALTH] = imax(0, E.P->inv[I_HEALTH] - amount);
  } else {
    Ent t = rd_ent(E, slot);
    t.health = (int8_t)imax(0, (int)t.health - amount);
    wr_ent(E, slot, t);
  }
}
CR_DEV void toward_player(const EnvRef &E, const Ent &e, bool long_axis, int &dx, int &dy) {
  int ox = E.P->ps[PS_PX] - e.x, oy = E.P->ps[PS_PY] - e.y;  // objects.py:54-62
  int ax = iabs(ox), ay = iabs(oy);
  if (long_axis ? ax > ay : ax <= ay) { dx = isign(ox); dy = 0; }
  else { dx = 0; dy = isign(oy); }
}
CR_DEV int dist_player(const EnvRef &E, const Ent &e) {  // objects.py:49-52
  return iabs(E.P->ps[PS_PX] - e.x) + iabs(E.P->ps[PS_PY] - e.y);
}
CR_DEV void random_dir(EnvRef &E, int &dx, int &dy) {  // objects.py:64-65
  int d = (int)rng_randint(E.rng, 4);
  dx = dir_x(d); dy = dir_y(d);
}

// ---- Player: objects.py:68-261 ---------------------------------------------------------------
CR_DEV void player_do_object(EnvRef &E, int slot) {  // objects.py:181-209
  PlayerS &P = *E.P;
  int dmg = 1;
  if (P.inv[I_WOOD_SWORD]) dmg = 2;
  if (P.inv[I_STONE_SWORD]) dmg = 3;
  if (P.inv[I_IRON_SWORD]) dmg = 5;
  Ent t = rd_ent(E, slot);
  if (t.type == T_PLANT) {
    if (t.aux > 300) {  // ripe, objects.py:401-403
      t.aux = 0;
      wr_ent(E, slot, t);
      P.inv[I_FOOD] += 4;
      P.ach[A_EAT_PLANT] += 1;
    }
  } else if (t.type == T_ZOMBIE || t.type == T_SKELETON || t.type == T_COW) {
    t.health = (int8_t)imax(0, (int)t.health - dmg);
    wr_ent(E, slot, t);
    if (t.health <= 0) {
      if (t.type == T_ZOMBIE) P.ach[A_DEFEAT_ZOMBIE] += 1;
      else if (t.type == T_SKELETON) P.ach[A_DEFEAT_SKELETON] += 1;
      else { P.inv[I_FOOD] += 6; P.ach[A_EAT_COW] += 1; P.ps[PS_HUNGER2] = 0; }
    }
  }
}
CR_DEV void player_do_material(EnvRef &E, int tx, int ty, int mat) {  // objects.py:211-229
  PlayerS &P = *E.P;
  if (mat == M_WATER) P.ps[PS_THIRST2] = 0;
  int req = -1, recv, ach, leaves;  // data.yaml:57-64
  double prob = 1.0;
  switch (mat) {
    case M_TREE: recv = I_WOOD; ach = A_COLLECT_WOOD; leaves = M_GRASS; break;
    case M_STONE: req = I_WOOD_PICKAXE; recv = I_STONE; ach = A_COLLECT_STONE; leaves = M_PATH; break;
    case M_COAL: req = I_WOOD_PICKAXE; recv = I_COAL; ach = A_COLLECT_COAL; leaves = M_PATH; break;
    case M_IRON: req = I_STONE_PICKAXE; recv = I_IRON; ach = A_COLLECT_IRON; leaves = M_PATH; break;
    case M_DIAMOND: req = I_IRON_PICKAXE; recv = I_DIAMOND; ach = A_COLLECT_DIAMOND; leaves = M_PATH; break;
    case M_WATER: recv = I_DRINK; ach = A_COLLECT_DRINK; leaves = M_WATER; break;
    case M_GRASS: recv = I_SAPLING; ach = A_COLLECT_SAPLING; leaves = M_GRASS; prob = 0.1; break;
    default: return;
  }
  if (req >= 0 && P.inv[req] < 1) return;
  wr_mat(E, tx, ty, leaves);
  if (rng_uniform(E.rng) <= prob) {  // drawn even when the probability is 1 (objects.py:226)
    P.inv[recv] += 1;
    P.ach[ach] += 1;
  }
}
CR_DEV void player_place(EnvRef &E, int which, int tx, int ty, int mat) {  // objects.py:231-247
  PlayerS &P = *E.P;
  int m2, slot;
  w_get(E, tx, ty, m2, slot);
  if (slot) return;
  int item, amount, result, ach;  // data.yaml:66-70
  unsigned where;
  switch (which) {
    case 0: item = I_STONE; amount = 1; result = M_STONE; ach = A_PLACE_STONE;
      where = WALKABLE | CR_MB(M_WATER) | CR_MB(M_LAVA); break;
    case 1: item = I_WOOD; amount = 2; result = M_TABLE; ach = A_PLACE_TABLE; where = WALKABLE; break;
    case 2: item = I_STONE; amount = 4; result = M_FURNACE; ach = A_PLACE_FURNACE; where = WALKABLE; break;
    default: item = I_SAPLING; amount = 1; result = -1; ach = A_PLACE_PLANT; where = CR_MB(M_GRASS); break;
  }
  if (mat == M_NONE || !((where >> mat) & 1u)) return;
  if (P.inv[item] < amount) return;
  P.inv[item] -= amount;
  if (result >= 0) {
    wr_mat(E, tx, ty, result);
  } else {  // Plant(world, target): health 1, grown 0 (objects.py:389-392)
    Ent p; p.type = T_PLANT; p.health = 1; p.x = (int16_t)tx; p.y = (int16_t)ty; p.aux = 0;
    w_add(E, p);
  }
  P.ach[ach] += 1;
}
CR_DEV void player_make(EnvRef &E, int which, const Ent &pl) {  // objects.py:249-261
  PlayerS &P = *E.P;
  const Geom &g = *E.g;
  unsigned nearby = 0;  // engine.py:95-103: numpy slice [x-1:x+2, y-1:y+2]; a negative start
  if (pl.x - 1 >= 0 && pl.y - 1 >= 0)  // wraps to an empty window (SURVEY.md Q7)
    for (int x = pl.x - 1; x <= pl.x + 1 && x < g.W; ++x)
      for (int y = pl.y - 1; y <= pl.y + 1 && y < g.H; ++y)
        nearby |= CR_MB(rd_mat(E, x, y));
  // data.yaml:72-78: wood_pickaxe, stone_pickaxe, iron_pickaxe, wood_sword, stone_sword, iron_sword
  int tier = which % 3;  // 0 wood, 1 stone, 2 iron
  int stone = tier == 1, coal = tier == 2, iron = tier == 2;
  if (!(nearby & CR_MB(M_TABLE))) return;
  if (tier == 2 && !(nearby & CR_MB(M_FURNACE))) return;
  if (P.inv[I_WOOD] < 1 || P.inv[I_STONE] < stone || P.inv[I_COAL] < coal || P.inv[I_IRON] < iron)
    return;
  P.inv[I_WOOD] -= 1; P.inv[I_STONE] -= stone; P.inv[I_COAL] -= coal; P.inv[I_IRON] -= iron;
  const int gives[6] = {I_WOOD_PICKAXE, I_STONE_PICKAXE, I_IRON_PICKAXE, I_WOOD_SWORD,
                        I_STONE_SWORD, I_IRON_SWORD};
  const int achs[6] = {A_MAKE_WOOD_PICKAXE, A_MAKE_STONE_PICKAXE, A_MAKE_IRON_PICKAXE,
                       A_MAKE_WOOD_SWORD, A_MAKE_STONE_SWORD, A_MAKE_IRON_SWORD};
  P.inv[gives[which]] += 1;
  P.ach[achs[which]] += 1;
}
CR_DEV void player_update(EnvRef &E, int action) {  // objects.py:99-131
  PlayerS &P = *E.P;
  Ent pl = rd_ent(E, 1);
  int tx = pl.x + dir_x(pl.aux), ty = pl.y + dir_y(pl.aux);
  int mat, slot;
  w_get(E, tx, ty, mat, slot);
  if (P.ps[PS_SLEEPING]) {
    if (P.inv[I_ENERGY] < 9) action = ACT_SLEEP;
    else { P.ps[PS_SLEEPING] = 0; P.ach[A_WAKE_UP] += 1; }
  }
  if (action >= ACT_LEFT && action <= ACT_DOWN) {  // objects.py:174-179
    pl.aux = (int16_t)(action - ACT_LEFT);
    obj_move(E, 1, pl, false, dir_x(pl.aux), dir_y(pl.aux), WALKABLE_PLAYER);
    wr_ent(E, 1, pl);
    if (rd_mat(E, pl.x, pl.y) == M_LAVA) P.inv[I_HEALTH] = 0;
  } else if (action == ACT_DO && slot) {
    player_do_object(E, slot);
  } else if (action == ACT_DO) {
    player_do_material(E, tx, ty, mat);
  } else if (action == ACT_SLEEP) {
    if (P.inv[I_ENERGY] < 9) P.ps[PS_SLEEPING] = 1;
  } else if (action >= ACT_PLACE_STONE && action <= ACT_PLACE_PLANT) {
    player_place(E, action - ACT_PLACE_STONE, tx, ty, mat);
  } else if (action >= ACT_MAKE_WOOD_PICKAXE && action <= ACT_MAKE_IRON_SWORD) {
    player_make(E, action - ACT_MAKE_WOOD_PICKAXE, pl);
  }
  const int sleeping = P.ps[PS_SLEEPING];
  // _update_life_stats, objects.py:133-152, in half units
  P.ps[PS_HUNGER2] += sleeping ? 1 : 2;
  if (P.ps[PS_HUNGER2] > 50) { P.ps[PS_HUNGER2] = 0; P.inv[I_FOOD] -= 1; }
  P.ps[PS_THIRST2] += sleeping ? 1 : 2;
  if (P.ps[PS_THIRST2] > 40) { P.ps[PS_THIRST2] = 0; P.inv[I_DRINK] -= 1; }
  if (sleeping) P.ps[PS_FATIGUE] = imin(P.ps[PS_FATIGUE] - 1, 0);
  else P.ps[PS_FATIGUE] += 1;
  if (P.ps[PS_FATIGUE] < -10) { P.ps[PS_FATIGUE] = 0; P.inv[I_ENERGY] += 1; }
  if (P.ps[PS_FATIGUE] > 30) { P.ps[PS_FATIGUE] = 0; P.inv[I_ENERGY] -= 1; }
  // _degen_or_regen_health, objects.py:154-167
  bool ok = P.inv[I_FOOD] > 0 && P.inv[I_DRINK] > 0 && (P.inv[I_ENERGY] > 0 || sleeping);
  if (ok) P.ps[PS_RECOVER2] += sleeping ? 4 : 2;
  else P.ps[PS_RECOVER2] -= sleeping ? 1 : 2;
  if (P.ps[PS_RECOVER2] > 50) { P.ps[PS_RECOVER2] = 0; P.inv[I_HEALTH] += 1; }
  if (P.ps[PS_RECOVER2] < -30) { P.ps[PS_RECOVER2] = 0; P.inv[I_HEALTH] = imax(0, P.inv[I_HEALTH] - 1); }
  for (int i = 0; i < N_ITEMS; ++i) P.inv[i] = imax(0, imin(P.inv[i], 9));  // objects.py:126-128
  // _wake_up_when_hurt, objects.py:169-172
  if (P.inv[I_HEALTH] < P.ps[PS_P_LAST_HEALTH]) P.ps[PS_SLEEPING] = 0;
  P.ps[PS_P_LAST_HEALTH] = P.inv[I_HEALTH];
  P.ps[PS_PX] = pl.x; P.ps[PS_PY] = pl.y;
}

// ---- creatures: objects.py:264-411 -----------------------------------------------------------
// Each returns with the record written back, or tombstoned when the object removed itself.
CR_DEV void entity_update(EnvRef &E, int slot) {
  Ent e = rd_ent(E, slot);
  bool removed = false;
  int dx, dy;
  switch (e.type) {
    case T_COW: {  // objects.py:274-279
      if (e.health <= 0) { wr_obj(E, e.x, e.y, 0); removed = true; }
      if (rng_uniform(E.rng) < 0.5) {
        random_dir(E, dx, dy);
        obj_move(E, slot, e, removed, dx, dy, WALKABLE);
      }
    } break;
    case T_ZOMBIE: {  // objects.py:294-312
      if (e.health <= 0) { wr_obj(E, e.x, e.y, 0); removed = true; }
      int dist = dist_player(E, e);
      if (dist <= 8 && rng_uniform(E.rng) < 0.9) {
        bool long_axis = rng_uniform(E.rng) < 0.8;
        toward_player(E, e, long_axis, dx, dy);
      } else {
        random_dir(E, dx, dy);
      }
      obj_move(E, slot, e, removed, dx, dy, WALKABLE);
      dist = dist_player(E, e);
      if (dist <= 1) {
        if (e.aux) {
          e.aux -= 1;
        } else {
          damage_slot(E, 1, E.P->ps[PS_SLEEPING] ? 7 : 2);
          e.aux = 5;
        }
      }
    } break;
    case T_SKELETON: {  // objects.py:327-351
      if (e.health <= 0) { wr_obj(E, e.x, e.y, 0); removed = true; }
      e.aux = (int16_t)imax(0, e.aux - 1);
      int dist = dist_player(E, e);
      bool done = false;
      if (dist <= 3) {
        bool long_axis = rng_uniform(E.rng) < 0.6;
        toward_player(E, e, long_axis, dx, dy);
        done = obj_move(E, slot, e, removed, -dx, -dy, WALKABLE);
      }
      if (done) {
      } else if (dist <= 5 && rng_uniform(E.rng) < 0.5) {  // _shoot, objects.py:343-351
        toward_player(E, e, true, dx, dy);
        if (e.aux <= 0 && (dx != 0 || dy != 0)) {
          int ax = e.x + dx, ay = e.y + dy;
          if (is_free(E, ax, ay, WALKABLE_ARROW)) {
            Ent a; a.type = T_ARROW; a.health = 0; a.x = (int16_t)ax; a.y = (int16_t)ay;
            a.aux = (int16_t)(dx < 0 ? 0 : dx > 0 ? 1 : dy < 0 ? 2 : 3);
            w_add(E, a);
            e.aux = 4;
          }
        }
      } else if (dist <= 8 && rng_uniform(E.rng) < 0.3) {
        bool long_axis = rng_uniform(E.rng) < 0.6;
        toward_player(E, e, long_axis, dx, dy);
        obj_move(E, slot, e, removed, dx, dy, WALKABLE);
      } else if (rng_uniform(E.rng) < 0.2) {
        random_dir(E, dx, dy);
        obj_move(E, slot, e, removed, dx, dy, WALKABLE);
      }
    } break;
    case T_ARROW: {  // objects.py:373-384
      dx = dir_x(e.aux); dy = dir_y(e.aux);
      int tx = e.x + dx, ty = e.y + dy, mat, hit;
      w_get(E, tx, ty, mat, hit);
      if (hit) {
        damage_slot(E, hit, 2);
        wr_obj(E, e.x, e.y, 0); removed = true;
      } else if (mat == M_NONE || !((WALKABLE_ARROW >> mat) & 1u)) {
        wr_obj(E, e.x, e.y, 0); removed = true;
        if (mat == M_TABLE || mat == M_FURNACE) wr_mat(E, tx, ty, M_PATH);
      } else {
        w_move(E, slot, e, tx, ty);
      }
    } break;
    case T_PLANT: {  // objects.py:405-411
      if (e.aux < 32767) e.aux += 1;  // grown; only `> 300` is ever observed
      bool hurt = false;
      for (int d = 0; d < 4; ++d) {
        int mat, s;
        w_get(E, e.x + dir_x(d), e.y + dir_y(d), mat, s);
        if (s) {
          int t = rd_ent(E, s).type;
          hurt = hurt || t == T_ZOMBIE || t == T_SKELETON || t == T_COW;
        }
      }
      if (hurt) e.health = (int8_t)imax(0, (int)e.health - 1);
      if (e.health <= 0) { wr_obj(E, e.x, e.y, 0); removed = true; }
    } break;
    default: return;
  }
  if (removed) e.type = T_NONE;
  wr_ent(E, slot, e);
}

// ---- order-preserving slot compaction (only relative order is semantic, engine.py:41-44) ----
CR_DEV void compact_slots(EnvRef &E, int lane) {
  const Geom &g = *E.g;
  int n = E.P->ps[PS_NSLOTS];
  int w = 1;
  for (int base = 1; base < n; base += CR_LANES) {
    int s = base + lane;
    Ent e; e.type = T_NONE;
    if (s < n) e = E.ents[s];
    bool live = e.type != T_NONE;
    uint32_t mask = cr_ballot(live);
    int dst = w + cr_popc(mask & cr_lanemask_lt(lane));
    if (live && dst != s) {
      E.ents[dst] = e;
      E.objmap[cell_of(g, e.x, e.y)] = (uint16_t)dst;
    }
    w += cr_popc(mask);
    cr_syncwarp();
  }
  if (lane == 0) E.P->ps[PS_NSLOTS] = w;
  cr_syncwarp();
}

// ---- balance: env.py:141-179 -------------------------------------------------------------------
// cnt layout per chunk: [0] grass cells, [1] path cells, [2] zombies, [3] skeletons, [4] cows.
// number of bytes of `w` equal to `b`
CR_DEV int cr_count_bytes_eq(uint32_t w, int b) {
#ifdef CR_HOSTSIM
  int n = 0;
  for (int k = 0; k < 4; ++k) n += (int)((w >> (8 * k)) & 0xFF) == b;
  return n;
#else
  return __popc(__vcmpeq4(w, 0x01010101u * (uint32_t)b)) >> 3;
#endif
}

// bit k of the result is set when byte k of `w` equals `b`
CR_DEV uint32_t cr_bytes_eq_mask(uint32_t w, int b) {
#ifdef CR_HOSTSIM
  uint32_t m = 0;
  for (int k = 0; k < 4; ++k) m |= (uint32_t)(((w >> (8 * k)) & 0xFF) == (uint32_t)b) << k;
  return m;
#else
  return ((__vcmpeq4(w, 0x01010101u * (uint32_t)b) & 0x08040201u) * 0x01010101u) >> 24;
#endif
}

// Grass / path cells of one 12-cell run of a map row (run r = x * ncy + cy); returns its chunk.
CR_DEV int census_run(const Geom &g, const uint8_t *mat, int r, bool words, int &grass, int &path) {
  const int x = r / g.ncy, cy = r - x * g.ncy;
  const uint8_t *row = mat + x * g.H + cy * CHUNK;
  const int len = imin(CHUNK, g.H - cy * CHUNK);
  grass = 0; path = 0;
  if (words) {
    const uint32_t *w = reinterpret_cast<const uint32_t *>(row);
#pragma unroll
    for (int k = 0; k < CHUNK / 4; ++k) {
      const uint32_t v = k * 4 < len ? w[k] : 0u;
      grass += cr_count_bytes_eq(v, M_GRASS);
      path += cr_count_bytes_eq(v, M_PATH);
    }
  } else {
#pragma unroll
    for (int y = 0; y < CHUNK; ++y) {
      int m = y < len ? row[y] : 0;
      grass += m == M_GRASS;
      path += m == M_PATH;
    }
  }
  return (x / CHUNK) * g.ncy + cy;
}

// Incremental census: recount one env from its terrain (after an install, or when the caller wrote
// `mat` itself).  All threads of the CTA; a block sync precedes (the terrain is in place) and
// follows (the counts are complete).
CR_DEV void census_recount(const Geom &g, const uint8_t *mat, int32_t *ccnt, int tid, int nthreads) {
  for (int i = tid; i < g.NCH * 2; i += nthreads) ccnt[i] = 0;
  cr_syncblock();
  const bool words = (g.H & 3) == 0;
  for (int r = tid; r < g.W * g.ncy; r += nthreads) {
    int grass, path;
    const int c = census_run(g, mat, r, words, grass, path);
    if (grass) cr_global_add(&ccnt[2 * c], grass);
    if (path) cr_global_add(&ccnt[2 * c + 1], path);
  }
  cr_syncblock();
}

// The same for the chunks of ONE chunk column (x / 12 == cx): nobody else writes their counts.
CR_DEV void census_recount_column(const Geom &g, const uint8_t *mat, int32_t *ccnt, int cx, int tid, int nthreads) {
  for (int i = tid; i < g.ncy * 2; i += nthreads) ccnt[cx * g.ncy * 2 + i] = 0;
  cr_syncblock();
  const bool words = (g.H & 3) == 0;
  const int x0 = cx * CHUNK, x1 = imin(x0 + CHUNK, g.W);
  for (int r = x0 * g.ncy + tid; r < x1 * g.ncy; r += nthreads) {
    int grass, path;
    const int c = census_run(g, mat, r, words, grass, path);
    if (grass) cr_global_add(&ccnt[2 * c], grass);
    if (path) cr_global_add(&ccnt[2 * c + 1], path);
  }
  cr_syncblock();
}

// Census of one env: creatures per (chunk, class) and grass / path cells per chunk.  The slot
// records are mirrored into shared memory on the way (rd_ent reads them there afterwards).
// `cnt` must be zeroed and synchronised by the caller; a block sync follows.  The first
// BAL_MEMBERS slots of every (chunk, class) pair are also noted (in arrival order, which is not
// slot order on the device) so that a despawn can name its creature without a slot scan.
constexpr int BAL_MEMBERS = 8;
constexpr int BAL_WC_STRIDE = 48;  // bytes per warp of balance_search's group counts

CR_DEV void balance_census(EnvRef &E, int tid, int nthreads, uint16_t *cnt, uint16_t *members,
                           int n_slots) {
  const Geom &g = *E.g;
  for (int s = 1 + tid; s < n_slots; s += nthreads) {
    Ent e = E.ents[s];
    if (s < ENT_SMEM) E.sents[s] = e;
    int cls = e.type == T_ZOMBIE ? 2 : e.type == T_SKELETON ? 3 : e.type == T_COW ? 4 : -1;
    if (cls >= 0) {
      const int c = chunk_of(g, e.x, e.y);
      const int pos = cr_smem_fetch_add(&cnt[c * 5 + cls], 1);
      if (pos < BAL_MEMBERS) members[(c * 3 + cls - 2) * BAL_MEMBERS + pos] = (uint16_t)s;
    }
  }
  if (g.incr_census) {  // the counts are kept current by wr_mat / wg_install_count
    for (int c = tid; c < g.NCH; c += nthreads) {
      if (E.ccnt[2 * c]) cr_smem_add(&cnt[c * 5 + 0], E.ccnt[2 * c]);
      if (E.ccnt[2 * c + 1]) cr_smem_add(&cnt[c * 5 + 1], E.ccnt[2 * c + 1]);
    }
    return;
  }
  const bool words = (g.H & 3) == 0;  // rows and 12-cell runs start on 4-byte boundaries
  for (int r = tid; r < g.W * g.ncy; r += nthreads) {  // one 12-cell run of a map row per thread
    int grass, path;
    const int c = census_run(g, E.mat, r, words, grass, path);
    if (grass) cr_smem_add(&cnt[c * 5 + 0], grass);
    if (path) cr_smem_add(&cnt[c * 5 + 1], path);
  }
}

// Decision of one (chunk, class) pair, env.py:157-179, evaluated by any lane (read-only on the
// world).  Returns 0 (nothing), BAL_SPAWN | type << 24 | cell, or BAL_DESPAWN | slot.  The
// occupancy test of a spawn is left to balance_apply because an earlier pair of the same tick may
// have filled the cell.  cls 0 zombie / grass, 1 skeleton / path, 2 cow / grass (env.py:143-155).
constexpr uint32_t BAL_SPAWN = 0x80000000u, BAL_DESPAWN = 0x40000000u, BAL_SEARCH = 0x20000000u;

CR_NOINLINE uint32_t balance_decide(const EnvRef &E, int chunk, int cls, int n, int space, double light,
                               int step, const uint16_t *members) {
  const Geom &g = *E.g;
  const int type = cls == 0 ? T_ZOMBIE : cls == 1 ? T_SKELETON : T_COW;
  const int material = cls == 1 ? M_PATH : M_GRASS;
  const int span = cls == 0 ? 6 : cls == 1 ? 7 : 5, despan = cls == 0 ? 0 : cls == 1 ? 7 : 5;
  const double p_spawn = cls == 0 ? 0.3 : cls == 1 ? 0.1 : 0.01;
  const double p_despawn = cls == 0 ? 0.4 : 0.1;
  int tmin, tmax;  // int() of the float targets (SURVEY.md Q13)
  if (cls == 0) { tmax = (int)(3.5 - 3 * light); tmin = space < 50 ? 0 : tmax; }
  else if (cls == 1) { tmin = space < 6 ? 0 : 1; tmax = 2; }
  else { tmin = space < 30 ? 0 : 1; tmax = (int)(1.5 + light); }
  if (n >= tmin && n <= tmax) return 0;  // neither branch draws
  Rng rng = rng_ctx((uint32_t)E.P->ps[PS_WORLD_SEED], D_BALANCE, (uint32_t)step, (uint32_t)chunk,
                    (uint32_t)cls);
  int cx = chunk / g.ncy, cy = chunk - cx * g.ncy;
  int xmin = cx * CHUNK, ymin = cy * CHUNK;
  int xmax = imin(xmin + CHUNK, g.W), ymax = imin(ymin + CHUNK, g.H);
  if (n < tmin && rng_uniform(rng) < p_spawn) {
    // xs[mask][i], ys[mask][i] with the mask in x-major order (env.py:166-169): WHICH cell that is takes
    // a scan of the chunk's 144 cells -- left to balance_search, a warp per spawn (this lane alone
    // made it the longest phase of the kernel)
    return BAL_SEARCH | rng_randint(rng, (uint32_t)space);
  } else if (n > tmax && rng_uniform(rng) < p_despawn) {
    int pick = (int)rng_randint(rng, (uint32_t)n), k = 0, last = E.P->ps[PS_NSLOTS];
    if (n <= BAL_MEMBERS) {  // creatures[pick] is the member with exactly `pick` smaller slots
      const uint16_t *m = members + (chunk * 3 + cls) * BAL_MEMBERS;
      int s = 0;
      for (int i = 0; i < n; ++i) {
        int rank = 0;
        for (int j = 0; j < n; ++j) rank += m[j] < m[i];
        if (rank == pick) s = m[i];
      }
      return dist_player(E, rd_ent(E, s)) >= despan ? (BAL_DESPAWN | (uint32_t)s) : 0u;
    }
    for (int s = 1; s < last; ++s) {  // crowded chunk: creatures[...] in slot order
      Ent e = rd_ent(E, s);
      if (e.type == type && chunk_of(g, e.x, e.y) == chunk && k++ == pick)
        return dist_player(E, e) >= despan ? (BAL_DESPAWN | (uint32_t)s) : 0u;
    }
  }
  return 0;
}

// The pick-th cell of `material` in chunk `job / 3`, x-major (env.py:166-169), by the lanes of one warp:
// every lane counts the matching cells of its 4-cell groups (12 rows x 3 groups), lane 0 walks the 36
// counts to the group that holds the pick and takes its bit; the decision replaces dec[job].
constexpr int BAL_GROUPS = CHUNK * (CHUNK / 4);
CR_DEV uint32_t balance_group_bits(const EnvRef &E, int x, int y0, int ymax, int material) {
  const Geom &g = *E.g;
  const uint8_t *p = E.mat + x * g.H + y0;
  if ((g.H & 3) == 0) {  // groups start on word boundaries and end on one (ymax too)
    return y0 < ymax ? cr_bytes_eq_mask(*reinterpret_cast<const uint32_t *>(p), material) : 0u;
  }
  uint32_t bits = 0;
  for (int k = 0; k < 4; ++k)
    if (y0 + k < ymax && p[k] == material) bits |= 1u << k;
  return bits;
}
CR_DEV void balance_search(const EnvRef &E, int job, int pick, int lane, uint8_t *wc, uint32_t *dec) {
  const Geom &g = *E.g;
  const int chunk = job / 3, cls = job - chunk * 3;
  const int type = cls == 0 ? T_ZOMBIE : cls == 1 ? T_SKELETON : T_COW;
  const int material = cls == 1 ? M_PATH : M_GRASS;
  const int span = cls == 0 ? 6 : cls == 1 ? 7 : 5;
  const int cx = chunk / g.ncy, cy = chunk - cx * g.ncy;
  const int xmin = cx * CHUNK, ymin = cy * CHUNK;
  const int xmax = imin(xmin + CHUNK, g.W), ymax = imin(ymin + CHUNK, g.H);
  int w_hit = -1, before = 0;  // the group that holds the pick, matching cells in the groups before it
#if CR_LANES >= 32
  // groups w = lane and (lanes 0..3) w = 32 + lane: inclusive prefix of their counts by shuffles, then
  // the first lane whose prefix exceeds the pick owns the group
  (void)wc;
  uint32_t bits[2];
  int inc[2];
  for (int h = 0; h < 2; ++h) {
    const int w = h * 32 + lane, xi = w / 3, k = w - xi * 3;
    bits[h] = w < BAL_GROUPS && xmin + xi < xmax ? balance_group_bits(E, xmin + xi, ymin + 4 * k, ymax, material) : 0u;
    int v = cr_popc(bits[h]);
    for (int d = 1; d < 32; d <<= 1) {
      const int u = (int)cr_shfl_up((uint32_t)v, d);
      if (lane >= d) v += u;
    }
    inc[h] = v;
  }
  const int total0 = (int)cr_shfl((uint32_t)inc[0], 31);
  const uint32_t m0 = cr_ballot(inc[0] > pick), m1 = cr_ballot(total0 + inc[1] > pick);
  const int h = m0 ? 0 : 1, owner = cr_ffs(m0 ? m0 : m1) - 1;  // space > pick: one of the two is non-empty
  if (lane == owner) {
    w_hit = h * 32 + lane;
    before = (h ? total0 : 0) + inc[h] - cr_popc(bits[h]);
  }
#else
  for (int w = lane; w < BAL_GROUPS; w += CR_LANES) {
    const int xi = w / 3, k = w - xi * 3;
    wc[w] = (uint8_t)(xmin + xi < xmax ? cr_popc(balance_group_bits(E, xmin + xi, ymin + 4 * k, ymax, material)) : 0);
  }
  cr_syncwarp();
  if (lane == 0) {
    int run = 0;
    for (int w = 0; w < BAL_GROUPS && w_hit < 0; ++w) {
      if (pick < run + wc[w]) { w_hit = w; before = run; }
      run += wc[w];
    }
  }
#endif
  if (w_hit >= 0) {  // one lane
    const int xi = w_hit / 3, k = w_hit - xi * 3;
    uint32_t group = balance_group_bits(E, xmin + xi, ymin + 4 * k, ymax, material);
    for (int q = before; q < pick; ++q) group &= group - 1;  // drop the lower set bits
    const int px = xmin + xi, py = ymin + 4 * k + cr_ffs(group) - 1;
    const bool away = iabs(E.P->ps[PS_PX] - px) + iabs(E.P->ps[PS_PY] - py) >= span;
    dec[job] = away ? (BAL_SPAWN | ((uint32_t)type << 24) | (uint32_t)cell_of(g, px, py)) : 0u;
  }
  cr_syncwarp();
}

// Applying the decisions (env.py:170-179) in (chunk, class) order, in parallel: a chunk's creatures and
// its spawn cells lie inside the chunk, so chunks only interact through the slot numbers of the spawns
// (append order, engine.py:54-55).  Every thread owns a contiguous range of chunks:
//   resolve  per chunk, its three decisions in class order: a despawn tombstones its creature at once; a
//            spawn is kept when its cell is empty NOW (`empty`, env.py:171: an earlier class of the
//            chunk may just have freed or taken it) -- kept spawns stay in dec[], the rest become 0
//   scan     exclusive prefix of the kept spawns over the threads' ranges -> first slot of each range
//   emit     the kept spawns take consecutive slots in decision order; beyond the capacity they are
//            dropped behind the sticky error bit, exactly like the serial w_add
CR_DEV int balance_resolve(EnvRef &E, uint32_t *dec, int c0, int c1) {
  int kept_total = 0;
  for (int c = c0; c < c1; ++c) {
    uint32_t taken[3];
    int kept = 0;
    for (int cls = 0; cls < 3; ++cls) {
      const uint32_t d = dec[c * 3 + cls];
      uint32_t keep = 0;
      if (d & BAL_DESPAWN) {
        const int s = (int)(d & 0xFFFFu);
        Ent e = rd_ent(E, s);
        wr_obj(E, e.x, e.y, 0);
        e.type = T_NONE;
        wr_ent(E, s, e);
      } else if (d & BAL_SPAWN) {
        const uint32_t cell = d & 0x00FFFFFFu;
        bool empty = E.objmap[cell] == 0;
        for (int j = 0; j < kept; ++j) empty = empty && taken[j] != cell;
        if (empty) { taken[kept++] = cell; keep = d; }
      }
      if (d) dec[c * 3 + cls] = keep;
    }
    kept_total += kept;
  }
  return kept_total;
}
CR_DEV void balance_emit(EnvRef &E, const uint32_t *dec, int c0, int c1, int slot) {
  const Geom &g = *E.g;
  for (int job = c0 * 3; job < c1 * 3; ++job) {
    const uint32_t d = dec[job];
    if (!d) continue;
    if (slot < g.CAP) {
      const int cell = (int)(d & 0x00FFFFFFu), type = (int)((d >> 24) & 0x3F);
      Ent o; o.type = (uint8_t)type; o.health = (int8_t)(type == T_ZOMBIE ? 5 : 3);
      o.x = (int16_t)(cell / g.H); o.y = (int16_t)(cell - (cell / g.H) * g.H); o.aux = 0;
      wr_ent(E, slot, o);
      E.objmap[cell] = (uint16_t)slot;
      const int ch = chunk_of(g, o.x, o.y);
      cr_smem_or(&E.stouched[ch >> 5], 1u << (ch & 31));
    }
    ++slot;
  }
}

// ---- env_balance: Env._balance_chunk for every ever-touched chunk (env.py:90-95,141-179) -------
// One CTA per env whose step is a multiple of 10 (k_balance), right after the tick.  All threads
// take the census, every (chunk, class) pair is decided by its own thread (draws are keyed per
// pair), thread 0 applies the rare spawns / despawns in reference order (sorted chunks; zombie,
// skeleton, cow).  `dec` holds NCH * 3 words.
CR_DEV void env_balance(const Geom &g, const State &st, const double *daylight_table, int env, int tid,
                        int nthreads, PlayerS *P, uint16_t *cnt, uint16_t *members, Ent *sents,
                        uint32_t *stouched, uint32_t *dec, int32_t *scan, uint8_t *wcount) {
  EnvRef E;
  E.g = &g;
  E.mat = st.mat + (size_t)env * g.NC;
  E.objmap = st.objmap + (size_t)env * g.NC;
  E.ents = st.ents + (size_t)env * g.CAP;
  E.touched = st.touched + (size_t)env * g.TW;
  E.P = P;
  E.sents = sents; E.stouched = stouched;
  E.ccnt = g.incr_census ? st.chunk_cnt + (size_t)env * g.NCH * 2 : nullptr;
  int32_t *ps_g = st.pstate + (size_t)env * PS_COUNT;
  for (int i = tid; i < PS_COUNT; i += nthreads) P->ps[i] = ps_g[i];
  for (int i = tid; i < g.NCH * 5; i += nthreads) cnt[i] = 0;
  for (int c = tid; c < g.TW; c += nthreads) stouched[c] = E.touched[c];
  if (tid == 0) cr_stamp(env, 0);
  const int n = ps_g[PS_NSLOTS], step = ps_g[PS_STEP];  // same words for every thread: one request
  const double daylight = daylight_table[imin(step, g.n_daylight - 1)];
  cr_syncblock();
  if (tid == 0) cr_stamp(env, 1);
  balance_census(E, tid, nthreads, cnt, members, n);
  cr_syncblock();
  if (tid == 0) cr_stamp(env, 2);
  for (int job = tid; job < g.NCH * 3; job += nthreads) {
    const int c = job / 3, cls = job - c * 3;
    uint32_t d = 0;
    if ((stouched[c >> 5] >> (c & 31)) & 1u) {  // only chunks that ever held an object
      const uint16_t *k = cnt + c * 5;
      d = balance_decide(E, c, cls, k[2 + cls], k[cls == 1 ? 1 : 0], daylight, step, members);
    }
    dec[job] = d;
  }
  cr_syncblock();
  {  // the spawns that passed their draw: a warp each finds the cell
    const int warp = tid / CR_LANES, lane = tid - warp * CR_LANES, nwarps = (nthreads + CR_LANES - 1) / CR_LANES;
    uint8_t *wc = wcount + warp * BAL_WC_STRIDE;
    for (int base = warp * CR_LANES; base < g.NCH * 3; base += nwarps * CR_LANES) {
      const int job = base + lane;
      const uint32_t d = job < g.NCH * 3 ? dec[job] : 0u;
      uint32_t mask = cr_ballot((d & BAL_SEARCH) != 0);
      while (mask) {
        const int b = cr_ffs(mask) - 1;
        mask &= mask - 1;
        balance_search(E, base + b, (int)(cr_shfl(d, b) & 0xFFFFu), lane, wc, dec);
      }
    }
  }
  cr_syncblock();
  if (tid == 0) cr_stamp(env, 3);
  const int per = (g.NCH + nthreads - 1) / nthreads;  // chunks per thread, contiguous: slot order == decision order
  const int c0 = imin(tid * per, g.NCH), c1 = imin(c0 + per, g.NCH);
  scan[tid] = balance_resolve(E, dec, c0, c1);
  cr_syncblock();
  if (tid == 0) {  // exclusive prefix over the threads' ranges (at most a few hundred words)
    int run = 0;
    for (int i = 0; i < nthreads; ++i) { const int v = scan[i]; scan[i] = run; run += v; }
    const int total = n + run;
    ps_g[PS_NSLOTS] = imin(total, g.CAP);
    ps_g[PS_ERROR] = P->ps[PS_ERROR] | (total > g.CAP ? ERR_SLOT_OVERFLOW : 0);
  }
  cr_syncblock();
  if (tid == 0) cr_stamp(env, 4);
  balance_emit(E, dec, c0, c1, n + scan[tid]);
  cr_syncblock();
  for (int c = tid; c < g.TW; c += nthreads) E.touched[c] = stouched[c];
  cr_syncblock();
  if (tid == 0) cr_stamp(env, 5);
}

// ---- the tick ---------------------------------------------------------------------------------
// Outputs reward/done and returns (on every lane) what the step still owes this env before its
// frame can be drawn: TICK_BALANCE on every 10th step (env.py:90-95), TICK_RESET when the episode
// ended and auto_reset is on (the caller regenerates it), both for a terminal step that also
// balances (only the terminal frame can tell; the state is discarded).
enum TickKind : int { TICK_FINAL = 0, TICK_BALANCE = 1, TICK_RESET = 2 };
constexpr int FS_LENGTH = 22, FS_DEAD = 23, FS_INV = 24, FS_POS = 40, FS_COUNT = 42;  // final_stats row
CR_DEV int env_step(const Geom &g, const State &st, const double *daylight_table, int env, int lane,
                     int action, PlayerS *P, Ent *sents, uint32_t *stouched, float *reward_out,
                     uint8_t *done_out, int auto_reset, int debug_skip = 0) {
  EnvRef E;
  E.g = &g;
  E.mat = st.mat + (size_t)env * g.NC;
  E.objmap = st.objmap + (size_t)env * g.NC;
  E.ents = st.ents + (size_t)env * g.CAP;
  E.touched = st.touched + (size_t)env * g.TW;
  E.P = P;
  E.ccnt = g.incr_census ? st.chunk_cnt + (size_t)env * g.NCH * 2 : nullptr;
  int32_t *inv_g = st.inventory + (size_t)env * N_ITEMS;
  int32_t *ach_g = st.achievements + (size_t)env * N_ACH;
  int32_t *ps_g = st.pstate + (size_t)env * PS_COUNT;
  if (lane == 0 && env < 4096) cr_stamp(8192 + env, 0);
  for (int i = lane; i < N_ITEMS; i += CR_LANES) P->inv[i] = inv_g[i];
  for (int i = lane; i < N_ACH; i += CR_LANES) P->ach[i] = ach_g[i];
  for (int i = lane; i < PS_COUNT; i += CR_LANES) P->ps[i] = ps_g[i];
  cr_syncwarp();

  if (P->ps[PS_NSLOTS] > g.CAP / 2) compact_slots(E, lane);
  E.sents = sents; E.stouched = stouched;
  if (lane < 2) grid_prefetch(E, P->ps[PS_PX] + (lane ? 2 : 0), P->ps[PS_PY]);  // player + make() window
  for (int s = lane; s < imin(P->ps[PS_NSLOTS], ENT_SMEM); s += CR_LANES) sents[s] = E.ents[s];
  for (int c = lane; c < g.TW; c += CR_LANES) stouched[c] = E.touched[c];
  const int step = P->ps[PS_STEP] + 1;  // env.py:84
  const int n0 = P->ps[PS_NSLOTS];      // snapshot of the slot list, engine.py:41-44
  const double daylight = daylight_table[imin(step, g.n_daylight - 1)];  // env.py:135-139
  if (step >= g.n_daylight && lane == 0) P->ps[PS_ERROR] |= ERR_DAYLIGHT_CLAMP;
  E.rng = rng_ctx((uint32_t)P->ps[PS_WORLD_SEED], D_UPDATE, (uint32_t)step);
  if (g.draw_prefetch) {
    // The k-th draw of the tick is Philox(key, counter = (k, step)) whatever happens before it, so
    // the first CR_LANES blocks cost one Philox in parallel instead of one each on lane 0's chain.
    for (int k = lane; k < DRAW_TAB; k += CR_LANES) {  // one iteration on the device
      const U4 o = philox4x32(E.rng.seed, D_UPDATE, (uint32_t)k, (uint32_t)step, 0, 0);
      P->draw[2 * k] = o.w[0];
      P->draw[2 * k + 1] = o.w[1];
    }
    E.rng.tab = P->draw;
    E.rng.ntab = DRAW_TAB;
  }
  cr_syncwarp();
  if (lane == 0 && env < 4096) cr_stamp(8192 + env, 1);
  if (lane == 0) {
    P->ps[PS_STEP] = step;
    // The player is slot 1 and its distance to itself is 0 < radius (env.py:87-89).
    player_update(E, action);
  }
  cr_syncwarp();
  if (lane == 0 && env < 4096) cr_stamp(8192 + env, 2);
  int traced_updates = 0;
  for (int base = 2; base < ((debug_skip & 2) ? 0 : n0); base += CR_LANES) {
    int s = base + lane;
    bool pred = false;
    if (s < n0) {
      Ent e = rd_ent(E, s);
      pred = e.type != T_NONE && dist_player(E, e) < g.radius;
      if (pred) grid_prefetch(E, e.x, e.y);
    }
    uint32_t mask = cr_ballot(pred);
    traced_updates += cr_popc(mask);
    if (lane == 0) {
      while (mask) {
        int b = cr_ffs(mask) - 1;
        mask &= mask - 1;
        entity_update(E, base + b);
      }
    }
    cr_syncwarp();
  }
  if (lane == 0 && env < 4096) { cr_stamp(8192 + env, 3); cr_stamp(8192 + env, 5, traced_updates); cr_stamp(8192 + env, 6, n0); }
  int kind = TICK_FINAL;
  uint32_t now = 0;  // achievements unlocked so far, one bit each (env.py:99-101), by all lanes
  for (int i = lane; i < N_ACH; i += CR_LANES) now |= (P->ach[i] > 0 ? 1u : 0u) << i;
  now = cr_reduce_or(now);
  if (lane == 0) {  // env.py:97-117
    int health = P->inv[I_HEALTH];
    double reward = (double)(health - P->ps[PS_LAST_HEALTH]) / 10;
    P->ps[PS_LAST_HEALTH] = health;
    uint32_t unlocked = (uint32_t)P->ps[PS_UNLOCKED];
    if (now & ~unlocked) { P->ps[PS_UNLOCKED] = (int32_t)(unlocked | now); reward += 1.0; }
    bool dead = health <= 0;
    bool over = g.length && step >= g.length;
    bool done = dead || over;
    reward_out[env] = (float)reward;  // info['reward']; the host zeroes it when reward=False
    done_out[env] = done ? 1 : 0;
    double *ret = st.ep_return + (size_t)env * 2;  // StatsRecorder bookkeeping, recorder.py:53-61
    const double total = ret[0] + reward;
    ret[0] = total;
    if (done) {
      ret[1] = total;
      // the terminal transition as the reference's info dict shows it (env.py:108-115); with
      // auto_reset the live rows already belong to the next episode when step() returns
      int32_t *fs = st.final_stats + (size_t)env * FS_COUNT;
      for (int i = 0; i < N_ACH; ++i) fs[i] = P->ach[i];
      fs[FS_LENGTH] = step;
      fs[FS_DEAD] = dead ? 1 : 0;  // terminated (health <= 0) vs truncated (length reached), env.py:105-107
      for (int i = 0; i < N_ITEMS; ++i) fs[FS_INV + i] = P->inv[i];
      fs[FS_POS] = P->ps[PS_PX]; fs[FS_POS + 1] = P->ps[PS_PY];
      if (st.final_world_seed) st.final_world_seed[env] = P->ps[PS_WORLD_SEED];  // before k_install replaces it
      P->ps[PS_EP_LENGTH] = step;
      if (auto_reset) kind |= TICK_RESET;
    }
    // Spawn / despawn balancing (env.py:90-95) runs in env_balance right after this tick; it
    // touches neither health nor achievements, so reward / done above are already final.
    if (step % 10 == 0 && !(debug_skip & 1)) kind |= TICK_BALANCE;
    // notes for the frame kernels: CTA order (frame_partition; a regenerated env starts by day) and which
    // envs k_view may prepare right away
    if (st.frame_night)
      st.frame_night[env] = (uint8_t)(((daylight < 0.5 && !(kind & TICK_RESET)) ? FRAME_NIGHT : 0) |
                                      (kind == TICK_FINAL ? FRAME_FINAL : 0));
  }
  cr_syncwarp();
  for (int c = lane; c < g.TW; c += CR_LANES) E.touched[c] = stouched[c];
  for (int i = lane; i < N_ITEMS; i += CR_LANES) inv_g[i] = P->inv[i];
  for (int i = lane; i < N_ACH; i += CR_LANES) ach_g[i] = P->ach[i];
  for (int i = lane; i < PS_COUNT; i += CR_LANES) ps_g[i] = P->ps[i];
  if (lane == 0 && env < 4096) cr_stamp(8192 + env, 4);
  return (int)cr_shfl((uint32_t)kind, 0);
}

// The step's work lists: envs to regenerate (k_install; they skip the balance, their state is
// discarded -- k_terminal balances them first when the terminal frame is wanted) and envs to balance
// (k_post).
CR_DEV void tick_to_lists(const State &st, int env, int kind) {
  if (kind & TICK_RESET) st.reset_list[cr_atomic_inc(st.reset_count)] = env;
  else if (kind & TICK_BALANCE) st.balance_list[cr_atomic_inc(st.balance_count)] = env;
}

}  // namespace cr
