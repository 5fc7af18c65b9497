// Trilinear hex geometry shared by the DG kernels (dg_facet_hex.cu, dg_transport_hex.cu): vertex v = (b0*2 + b1)*2
// + b2 of a cell sits at reference point (b0, b1, b2); X holds the 8 vertices' coordinates, 3 per vertex.
#pragma once

// the inverse Jacobian K[d][c] = dxi_d/dx_c and |det J| of the cell's trilinear map at reference point xi
__device__ __forceinline__ double trilinear_inverse_jacobian(const double *X, const double xi[3], double K[3][3])
{
    double J[3][3];
#pragma unroll
    for (int c = 0; c < 3; c++)
#pragma unroll
        for (int d = 0; d < 3; d++) J[c][d] = 0.0;
#pragma unroll
    for (int v = 0; v < 8; v++) {
        const int b0 = (v >> 2) & 1, b1 = (v >> 1) & 1, b2 = v & 1;
        const double f0 = b0 ? xi[0] : 1.0 - xi[0], f1 = b1 ? xi[1] : 1.0 - xi[1], f2 = b2 ? xi[2] : 1.0 - xi[2];
        const double g0 = (b0 ? 1.0 : -1.0) * f1 * f2;
        const double g1 = (b1 ? 1.0 : -1.0) * f0 * f2;
        const double g2 = (b2 ? 1.0 : -1.0) * f0 * f1;
#pragma unroll
        for (int c = 0; c < 3; c++) {
            const double xc = X[v * 3 + c];
            J[c][0] = fma(xc, g0, J[c][0]);
            J[c][1] = fma(xc, g1, J[c][1]);
            J[c][2] = fma(xc, g2, J[c][2]);
        }
    }
    const double A00 = J[1][1] * J[2][2] - J[1][2] * J[2][1];
    const double A01 = J[0][2] * J[2][1] - J[0][1] * J[2][2];
    const double A02 = J[0][1] * J[1][2] - J[0][2] * J[1][1];
    const double det = J[0][0] * A00 + J[1][0] * A01 + J[2][0] * A02;
    const double r = 1.0 / det;
    K[0][0] = A00 * r;
    K[0][1] = A01 * r;
    K[0][2] = A02 * r;
    K[1][0] = (J[1][2] * J[2][0] - J[1][0] * J[2][2]) * r;
    K[1][1] = (J[0][0] * J[2][2] - J[0][2] * J[2][0]) * r;
    K[1][2] = (J[0][2] * J[1][0] - J[0][0] * J[1][2]) * r;
    K[2][0] = (J[1][0] * J[2][1] - J[1][1] * J[2][0]) * r;
    K[2][1] = (J[0][1] * J[2][0] - J[0][0] * J[2][1]) * r;
    K[2][2] = (J[0][0] * J[1][1] - J[0][1] * J[1][0]) * r;
    return fabs(det);
}

// the trilinear interpolant at xi of a field F given at the 8 vertices (3 values per vertex)
__device__ __forceinline__ void trilinear_interpolate(const double *F, const double xi[3], double out[3])
{
    out[0] = out[1] = out[2] = 0.0;
#pragma unroll
    for (int v = 0; v < 8; v++) {
        const double w = ((v >> 2) & 1 ? xi[0] : 1.0 - xi[0]) * ((v >> 1) & 1 ? xi[1] : 1.0 - xi[1]) *
                         (v & 1 ? xi[2] : 1.0 - xi[2]);
#pragma unroll
        for (int c = 0; c < 3; c++) out[c] = fma(w, F[v * 3 + c], out[c]);
    }
}
