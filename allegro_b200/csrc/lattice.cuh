// The inverse of a lattice, computed once on the host for every kernel that works in fractional coordinates
// (nl_lattice_geom in nlist.cu, ab2_slab_plan_count_lattice in slab_md.cu).  data._lattice_metrics mirrors these
// operations in the same order, so the host and the device agree on every quotient.
#pragma once
#include <cmath>

struct Ab2Lattice {
    double h[3][3];     // rows: h[a] = lattice vector a
    double hinv[3][3];  // h^-1: f = pos . hinv
    double cr[3][3];    // cr[a] = h[a+1] x h[a+2] = det . (column a of hinv)
    double det;
};

// rows [9] -> lat.  1: a row is not finite; 2: singular (or rows within 1e-12 rad of a common plane); 0: ok
inline int ab2_lattice_inverse(const double* rows, Ab2Lattice& lat) {
    for (int k = 0; k < 9; ++k) {
        if (!std::isfinite(rows[k])) return 1;
        lat.h[k / 3][k % 3] = rows[k];
    }
    double norm[3];
    for (int a = 0; a < 3; ++a) {
        const double* p = lat.h[(a + 1) % 3];
        const double* q = lat.h[(a + 2) % 3];
        lat.cr[a][0] = p[1] * q[2] - p[2] * q[1];
        lat.cr[a][1] = p[2] * q[0] - p[0] * q[2];
        lat.cr[a][2] = p[0] * q[1] - p[1] * q[0];
        norm[a] = std::sqrt(lat.h[a][0] * lat.h[a][0] + lat.h[a][1] * lat.h[a][1] + lat.h[a][2] * lat.h[a][2]);
    }
    lat.det = lat.h[0][0] * lat.cr[0][0] + lat.h[0][1] * lat.cr[0][1] + lat.h[0][2] * lat.cr[0][2];
    if (!std::isfinite(lat.det) || !(std::fabs(lat.det) > 1e-12 * norm[0] * norm[1] * norm[2])) return 2;
    for (int a = 0; a < 3; ++a)
        for (int x = 0; x < 3; ++x) lat.hinv[x][a] = lat.cr[a][x] / lat.det;
    return 0;
}

// H_a = |det| / |h[a+1] x h[a+2]|: the height of the cell along axis a (the distance between its two faces)
inline double ab2_lattice_height(const Ab2Lattice& lat, int a) {
    const double* c = lat.cr[a];
    return std::fabs(lat.det) / std::sqrt(c[0] * c[0] + c[1] * c[1] + c[2] * c[2]);
}
