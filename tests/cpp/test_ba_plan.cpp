// The bundle-adjustment structure planner (lvio_fusion_b200/csrc/ba_plan.h) on its own, without a GPU (tests/test_ba_plan.py).
//
//   test_ba_plan problem IN OUT      IN: the flat problem of tests/shim_util.py::dump_ba, optionally followed by the constant flags
//                                    (np + nv + nr bytes).  Runs plan_ba (132 SMs, one rank) and writes the plan as named int64
//                                    arrays: int32 name length, name, int64 count, count x int64.  A planner error prints
//                                    "error <code> <message>" and exits with 3.
//   test_ba_plan band N BAND NO_TREE plan_reduced_solver on the envelope of a full band; prints levels, wide, chol_smem.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <string>
#include <vector>
#include "../../lvio_fusion_b200/csrc/ba_plan.h"

using namespace lvb;

static const int kSmCount = 132;

template <class T> static bool read_n(FILE* f, std::vector<T>& v, size_t n) { v.resize(n); return fread(v.data(), sizeof(T), n, f) == n; }

struct Writer {
    FILE* f;
    template <class T> void put(const char* name, const T* v, size_t n) {
        const int len = (int)strlen(name);
        const long long cnt = (long long)n;
        fwrite(&len, 4, 1, f); fwrite(name, 1, len, f); fwrite(&cnt, 8, 1, f);
        for (size_t i = 0; i < n; ++i) { const long long x = (long long)v[i]; fwrite(&x, 8, 1, f); }
    }
    template <class T> void put(const char* name, const std::vector<T>& v) { put(name, v.data(), v.size()); }
    void scalar(const char* name, long long x) { put(name, &x, 1); }
};

static int problem(const char* in_path, const char* out_path) {
    FILE* f = fopen(in_path, "rb");
    if (!f) { perror(in_path); return 2; }
    std::vector<int32_t> head;
    if (!read_n(f, head, 10)) { fprintf(stderr, "short header\n"); return 2; }
    const int np = head[0], nv = head[1], nr = head[2];
    std::vector<double> skip, fc[6];
    std::vector<int32_t> fi[6];
    bool ok = read_n(f, skip, 22) && read_n(f, skip, (size_t)7 * np) && read_n(f, skip, (size_t)3 * nv) && read_n(f, skip, (size_t)nr);
    BaProblemView in;
    in.np = np; in.nv = nv; in.nr = nr;
    for (int k = 0; k < 6 && ok; ++k) {
        in.n[k] = head[3 + k];
        if (in.n[k]) ok = read_n(f, fc[k], (size_t)in.n[k] * kConstStride[k]) && read_n(f, fi[k], (size_t)in.n[k] * kIdxStride[k]);
        in.fc[k] = fc[k].data(); in.fi[k] = fi[k].data();
    }
    if (!ok) { fprintf(stderr, "short problem file\n"); return 2; }
    std::vector<uint8_t> cflags((size_t)np + nv + nr, 0);
    const size_t got = fread(cflags.data(), 1, cflags.size(), f);
    fclose(f);
    if (got != 0 && got != cflags.size()) { fprintf(stderr, "short constant flags\n"); return 2; }
    in.pose_const = cflags.data(); in.vec3_const = cflags.data() + np; in.rho_const = cflags.data() + np + nv;

    BaPlan p;
    std::string err;
    std::vector<std::string> phases;
    PlanHooks hooks;
    hooks.phase_done = [&](const char* name) { phases.push_back(name); };
    const int rc = plan_ba(in, kSmCount, 1, false, false, hooks, p, err);
    if (rc != LVB_OK) { printf("error %d %s\n", rc, err.c_str()); return 3; }
    for (const std::string& s : phases) printf("phase %s\n", s.c_str());

    Writer w{fopen(out_path, "wb")};
    if (!w.f) { perror(out_path); return 2; }
    static const char* kOrder[6] = {"order0", "order1", "order2", "order3", "order4", "order5"};
    for (int k = 0; k < 6; ++k) w.put(kOrder[k], p.order[k]);
    w.put("nd", p.nd, 6);
    w.put("pose_off", p.pose_off); w.put("vec3_off", p.vec3_off); w.put("rho_slot", p.rho_slot); w.put("canon", p.canon);
    w.put("lm_start", p.lm_start); w.put("lm_fac", p.lm_fac); w.put("tf_slot", p.tf_slot);
    w.put("sw_group", p.sw_group); w.put("sw_lm", p.sw_lm); w.put("grp_ns", p.grp_ns); w.put("grp_off", p.grp_off);
    w.put("chol_rmax", p.chol_rmax); w.put("chol_cmin", p.chol_cmin);
    w.put("tc_cdim", p.tc_cdim); w.put("tc_off", p.tc_off);
    w.scalar("dimc", p.dimc); w.scalar("n_pose_free", p.n_pose_free); w.scalar("n_vec3_free", p.n_vec3_free); w.scalar("n_rho_free", p.n_rho_free);
    w.scalar("n_schur_warps", p.n_schur_warps); w.scalar("schur_cols_max", p.schur_cols_max);
    w.scalar("band", p.band); w.scalar("true_band", p.true_band); w.scalar("dense", p.dense); w.scalar("srow", p.srow); w.scalar("soff", p.soff);
    w.scalar("nS", (long long)p.nS); w.scalar("solvable", p.solvable); w.scalar("tc_ok", p.tc_ok);
    w.scalar("tree_levels", p.solver.tree_levels); w.scalar("wide", p.solver.wide); w.scalar("chol_smem", (long long)p.solver.chol_smem);
    w.scalar("max_cta_smem", MAX_CTA_SMEM);
    fclose(w.f);
    return 0;
}

int main(int argc, char** argv) {
    if (argc == 4 && !strcmp(argv[1], "problem")) return problem(argv[2], argv[3]);
    if (argc == 5 && !strcmp(argv[1], "band")) {
        const int n = atoi(argv[2]), band = atoi(argv[3]);
        std::vector<int> rmax, cmin;
        uniform_band_envelope(n, band, rmax, cmin);
        const SolverPlan s = plan_reduced_solver(n, band, band - 31, rmax, kSmCount, atoi(argv[4]) != 0);
        printf("%d %d %zu %d\n", s.tree_levels, (int)s.wide, s.chol_smem, (int)MAX_CTA_SMEM);
        return 0;
    }
    fprintf(stderr, "usage: test_ba_plan problem IN OUT | band N BAND NO_TREE\n");
    return 2;
}
