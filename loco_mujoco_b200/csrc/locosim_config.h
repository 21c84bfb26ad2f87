// Compile-time configurations: one step-kernel instantiation per (friction cone, integrator) family.
// NV / NB / NG / MAXOBS are capacities (model sizes must be <=), MAXCON / MAXROW bound the active contact set.
// CONE: 0 pyramidal, 1 elliptic (mjModel.opt.cone); RK4: 0 Euler, 1 RK4 (mjModel.opt.integrator).
// CONVEX: 1 = the configuration carries the general convex (mjc_Convex / MPR) narrow phase; models with such pairs need it.
// BOXBOX: 1 = it also carries the exact edge-edge branch of mjc_BoxBox; models with box-box pairs need it (A1, Talos, H1 have none:
//         their kernels stay free of that code - an A/B on one box showed -1 % for A1 from its mere presence).
// HULL: 1 = its convex phase runs the capsule-hull test on pairs with flag 4 (sphere | capsule | cylinder vs cylinder) after
//       the box test, and skips the block's job queue when no env has a job (UnitreeA1: every job was such a near miss).
//       An optimisation only: with 0 those pairs go on to MPR, and the kernels of the other configurations keep the code
//       they had without it.
// PRIMLEAN: 1 = the primitive pairs are filtered in one lean pass (two pairs per lane per trip, hits compacted in pair
//           order) and the narrow phase runs once over the compacted hits in sets of 32, instead of a narrow round after
//           every round of 32 filtered pairs (UnitreeA1: only its 37 floor pairs of 357 ever pass). Same contact list bit
//           for bit; with 0 the kernels keep the round loop only. UnitreeA1's flag is the macro LOCOSIM_PRIMLEAN (default 1),
//           so that a build with -DLOCOSIM_PRIMLEAN=0 shows what the lean pass costs in registers and stack.
// TERRAIN: 1 = collision() ends with the height-field pass (locosim_core.cuh terrain_pass): the pairs (terrain, g) of a
//          model with a terrain. Compiled only in locosim_terrain.cu (and the serial build), so the kernels of every other
//          configuration keep their code.
// The two 31-dof configurations serve the full-body variants (arms, and for Atlas the back joint): their models collide with
// the floor only, so they carry no box-box branch; they keep the convex narrow phase that every other configuration carries,
// so that their collision code is the one every bundled model already runs.
#pragma once
#ifndef LOCOSIM_PRIMLEAN
#define LOCOSIM_PRIMLEAN 1
#endif
struct CfgEllEuler { enum { NV = 18, NB = 14, NG = 40,  MAXCON = 16, MAXROW = 64, MAXOBS = 64, CONE = 1, RK4 = 0, CONVEX = 1, BOXBOX = 0, HULL = 1, PRIMLEAN = LOCOSIM_PRIMLEAN, TERRAIN = 0 }; };  // UnitreeA1
struct CfgPyrEuler { enum { NV = 18, NB = 14, NG = 56,  MAXCON = 16, MAXROW = 64, MAXOBS = 64, CONE = 0, RK4 = 0, CONVEX = 1, BOXBOX = 0, HULL = 0, PRIMLEAN = 0, TERRAIN = 0 }; };  // Talos, UnitreeH1
struct CfgPyrRK4   { enum { NV = 19, NB = 12, NG = 100, MAXCON = 16, MAXROW = 64, MAXOBS = 64, CONE = 0, RK4 = 1, CONVEX = 1, BOXBOX = 1, HULL = 0, PRIMLEAN = 0, TERRAIN = 0 }; };  // Atlas, HumanoidTorque
struct CfgPyrEuler29 { enum { NV = 29, NB = 26, NG = 48,  MAXCON = 16, MAXROW = 64, MAXOBS = 64, CONE = 0, RK4 = 0, CONVEX = 1, BOXBOX = 1, HULL = 0, PRIMLEAN = 0, TERRAIN = 0 }; };  // UnitreeG1 (29 dofs <= 32 lanes)
struct CfgPyrRK4_31 { enum { NV = 31, NB = 27, NG = 100, MAXCON = 16, MAXROW = 64, MAXOBS = 72, CONE = 0, RK4 = 1, CONVEX = 1, BOXBOX = 0, HULL = 0, PRIMLEAN = 0, TERRAIN = 0 }; };  // Atlas with arms (+ back)
struct CfgPyrEuler31 { enum { NV = 31, NB = 26, NG = 52,  MAXCON = 16, MAXROW = 64, MAXOBS = 72, CONE = 0, RK4 = 0, CONVEX = 1, BOXBOX = 0, HULL = 0, PRIMLEAN = 0, TERRAIN = 0 }; };  // Talos with arms
// UnitreeA1 on a height field: CfgEllEuler with the terrain pass (same EnvS, same envs per SM)
struct CfgEllEulerTerrain { enum { NV = 18, NB = 14, NG = 40,  MAXCON = 16, MAXROW = 64, MAXOBS = 64, CONE = 1, RK4 = 0, CONVEX = 1, BOXBOX = 0, HULL = 1, PRIMLEAN = LOCOSIM_PRIMLEAN, TERRAIN = 1 }; };
