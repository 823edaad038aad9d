// Native receding-horizon loop on libomgb200.so: the C++ twin of a deployed controller calling the
// reference's exported Point2Point::update() (omgtools/export/point2point/Point2Point.cpp:119-205)
// for B independent instances at once.  The deployable artefacts are a table file
// (omg_tools_b200.solver.b200.save_tables) and an MPC file (save_mpc for a fixed horizon,
// save_mpc_freeT for a free motion time; the example reads either); no Python and no CasADi at
// run time.
//
//   g++ -O2 -I include examples/native/native_mpc.cpp -o native_mpc \
//       -L omg_tools_b200/csrc -lomgb200 -Wl,-rpath,$PWD/omg_tools_b200/csrc
//   ./native_mpc problem.omgtbl problem.omgmpc B N trajectory_length ideal|integrate \
//       state0.f64 stateT.f64 obstacles.f64 traj_out.f64 [problem.omgobs shapes.f64 avoid.i32]
//
// state0.f64 / stateT.f64: B rows of n_dim doubles; obstacles.f64: B rows of n_obs records
// {x, v, a, theta} of 3 n_dim + 1 doubles (an empty file without obstacles).  This example holds
// the goal and the obstacles fixed and feeds the first sample of each returned plan back as the
// measured state, as if the vehicle followed its plan exactly; a real caller passes what its
// sensors measure.  traj_out.f64 receives, per update, the state and then the input trajectories
// [B][trajectory_length][n_dim].
//
// With the three optional arguments the example also drives the rest of the reference's obstacle_t:
// problem.omgobs is the obstacle file (save_mpc_obstacles), shapes.f64 holds B rows of the obstacles'
// checkpoints and radii (per obstacle its chk_len checkpoint coordinates, then its rad_len radii) and
// avoid.i32 B rows of n_obs int32 avoid flags.  They are set before the first update, and at update
// N / 2 every avoid flag is flipped, as a caller does when an obstacle starts or stops mattering.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "omg_b200.h"

static bool read_doubles(const char* path, std::vector<double>& v) {
  FILE* fp = fopen(path, "rb");
  if (!fp) return false;
  const size_t got = v.empty() ? 0 : fread(v.data(), sizeof(double), v.size(), fp);
  fclose(fp);
  return got == v.size();
}

int main(int argc, char** argv) {
  if (argc != 11 && argc != 14) {
    fprintf(stderr, "usage: %s tables mpc B N trajectory_length ideal|integrate state0 stateT obstacles traj_out "
            "[obstacle_file shapes avoid]\n", argv[0]);
    return 2;
  }
  omg_tables* tb = omg_tables_read(argv[1]);
  if (!tb) { fprintf(stderr, "tables: %s\n", omg_last_error()); return 1; }
  // a fixed-horizon MPC file, else a free-T one
  omg_mpc_desc* desc = omg_mpc_read(argv[2]);
  omg_mpc_freeT_desc* fdesc = desc ? nullptr : omg_mpc_freet_read(argv[2]);
  if (!desc && !fdesc) { fprintf(stderr, "mpc: %s\n", omg_last_error()); return 1; }
  const int B = atoi(argv[3]), N = atoi(argv[4]), tl = atoi(argv[5]);
  const int nd = desc ? desc->n_dim : fdesc->n_dim, n_obs = desc ? desc->n_obs : fdesc->n_obs;
  const int mode = strcmp(argv[6], "integrate") == 0 ? OMG_MPC_PREDICT_INTEGRATE : OMG_MPC_PREDICT_IDEAL;
  std::vector<double> state0((size_t)B * nd), stateT((size_t)B * nd), obs((size_t)B * n_obs * (3 * nd + 1));
  if (!read_doubles(argv[7], state0) || !read_doubles(argv[8], stateT) || !read_doubles(argv[9], obs)) {
    fprintf(stderr, "bad input files\n"); return 1;
  }
  omg_options opt;
  omg_default_options(&opt);
  omg_problem* h = omg_problem_create(tb, &opt, 0);
  if (!h) { fprintf(stderr, "create: %s\n", omg_last_error()); return 1; }
  omg_mpc* mpc = desc ? omg_mpc_create(h, desc, B, tl, mode) : omg_mpc_create_freet(h, fdesc, B, tl, mode);
  if (!mpc) { fprintf(stderr, "mpc create: %s\n", omg_last_error()); return 1; }
  omg_mpc_obstacles_desc* odesc = nullptr;
  std::vector<int32_t> avoid;
  if (argc == 14) {
    odesc = omg_mpc_obstacles_read(argv[11]);
    if (!odesc) { fprintf(stderr, "obstacles: %s\n", omg_last_error()); return 1; }
    size_t n_shape = 0;
    for (int k = 0; k < odesc->n_obs; ++k) n_shape += (size_t)odesc->chk_len[k] + odesc->rad_len[k];
    std::vector<double> shapes((size_t)B * n_shape);
    avoid.resize((size_t)B * n_obs);
    FILE* fa = fopen(argv[13], "rb");
    const bool got = fa && (avoid.empty() || fread(avoid.data(), 4, avoid.size(), fa) == avoid.size());
    if (fa) fclose(fa);
    if (!read_doubles(argv[12], shapes) || !got) { fprintf(stderr, "bad obstacle input files\n"); return 1; }
    if (omg_mpc_attach_obstacles(mpc, odesc) != 0 || omg_mpc_set_obstacles_host(mpc, shapes.data(), avoid.data()) != 0) {
      fprintf(stderr, "obstacles: %s\n", omg_last_error()); return 1;
    }
  }
  std::vector<double> xtraj((size_t)B * tl * nd, 0.0), utraj((size_t)B * tl * nd, 0.0);
  std::vector<int32_t> status(B), iters(B);
  FILE* fo = fopen(argv[10], "wb");
  if (!fo) { fprintf(stderr, "cannot write %s\n", argv[10]); return 1; }
  for (int k = 0; k < N; ++k) {
    if (odesc && k == N / 2) {        // flip every avoid flag from this update on
      for (int32_t& a : avoid) a = !a;
      if (omg_mpc_set_obstacles_host(mpc, nullptr, avoid.data()) != 0) {
        fprintf(stderr, "obstacles: %s\n", omg_last_error()); return 1;
      }
    }
    if (omg_mpc_update_host(mpc, state0.data(), stateT.data(), obs.data(), xtraj.data(), utraj.data(),
                            status.data(), iters.data()) != 0) {
      fprintf(stderr, "update: %s\n", omg_last_error()); return 1;
    }
    for (int b = 0; b < B; ++b) {
      printf("update %d instance %d status %d iters %d\n", k, b, status[b], iters[b]);
      // a failed instance keeps its state: Point2Point::update returned false, the caller may recover;
      // a stopped one (free motion time, OMG_MPC_STOPPED) has arrived
      if (status[b] == OMG_SOLVE_SUCCEEDED)
        for (int c = 0; c < nd; ++c) state0[(size_t)b * nd + c] = xtraj[(size_t)b * tl * nd + c];
    }
    fwrite(xtraj.data(), sizeof(double), xtraj.size(), fo);
    fwrite(utraj.data(), sizeof(double), utraj.size(), fo);
  }
  fclose(fo);
  omg_mpc_destroy(mpc);
  omg_problem_destroy(h);
  omg_mpc_free_desc(desc);
  omg_mpc_freet_release(fdesc);
  omg_mpc_obstacles_release(odesc);
  omg_tables_free(tb);
  return 0;
}
