// The single-CTA storage choice of plan_reduced_solver (lvio_fusion_b200/csrc/ba_plan.h) without a GPU (tests/test_ba_plan_resident.py).
//
//   test_ba_plan_resident problem IN      IN: the flat problem of tests/shim_util.py::dump_ba.  Runs plan_ba (132 SMs, one rank) and
//                                         prints "dimc resident resident_smem max_cta_smem tree_levels wide" and then the envelope
//                                         rmax of every 32-column step on a second line.  A planner error prints "error <code> <message>"
//                                         and exits with 3.
//   test_ba_plan_resident band N BAND NO_TREE  plan_reduced_solver on the envelope of a full band; prints resident, resident_smem,
//                                         max_cta_smem.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <string>
#include <vector>
#include "../../lvio_fusion_b200/csrc/ba_plan.h"

using namespace lvb;

static const int kSmCount = 132;

template <class T> static bool read_n(FILE* f, std::vector<T>& v, size_t n) { v.resize(n); return fread(v.data(), sizeof(T), n, f) == n; }

static int problem(const char* in_path) {
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
    fclose(f);
    if (!ok) { fprintf(stderr, "short problem file\n"); return 2; }
    std::vector<uint8_t> cflags((size_t)np + nv + nr, 0);
    in.pose_const = cflags.data(); in.vec3_const = cflags.data() + np; in.rho_const = cflags.data() + np + nv;
    BaPlan p;
    std::string err;
    const int rc = plan_ba(in, kSmCount, 1, false, false, PlanHooks{}, p, err);
    if (rc != LVB_OK) { printf("error %d %s\n", rc, err.c_str()); return 3; }
    printf("%d %d %zu %d %d %d\n", p.dimc, (int)p.solver.resident, p.solver.resident_smem, (int)MAX_CTA_SMEM, p.solver.tree_levels, (int)p.solver.wide);
    for (int s = 0; s < (p.dimc + 31) / 32; ++s) printf("%s%d", s ? " " : "", p.chol_rmax[s]);
    printf("\n");
    return 0;
}

int main(int argc, char** argv) {
    if (argc == 3 && !strcmp(argv[1], "problem")) return problem(argv[2]);
    if (argc == 5 && !strcmp(argv[1], "band")) {
        const int n = atoi(argv[2]), band = atoi(argv[3]);
        std::vector<int> rmax, cmin;
        uniform_band_envelope(n, band, rmax, cmin);
        const SolverPlan s = plan_reduced_solver(n, band, band - 31, rmax, kSmCount, atoi(argv[4]) != 0);
        printf("%d %zu %d\n", (int)s.resident, s.resident_smem, (int)MAX_CTA_SMEM);
        return 0;
    }
    fprintf(stderr, "usage: test_ba_plan_resident problem IN | band N BAND NO_TREE\n");
    return 2;
}
