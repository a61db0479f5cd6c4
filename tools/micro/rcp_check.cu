// Does MUFU.RCP return exactly 1 for 1, and MUFU.EX2 exactly 1 for -0?  The paired blend backward relies on it: a masked
// pixel's transmittance is kept only because T * rcp.approx(1 - 0) == T.  nvcc -arch=sm_90a -o rcp_check rcp_check.cu && ./rcp_check
#include <cstdio>
#include <cstring>
__global__ void k(float *out, float one, float nzero) {
    float r, e;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(one));
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(nzero));
    out[0] = r; out[1] = e;
    // every power of two and a sweep of other inputs: relative error of rcp.approx
    float worst = 0.f;
    for (int i = 0; i < 1 << 20; ++i) {
        float x = 1.0f + (float)i * (1.0f / (1 << 20)), y;
        asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
        float err = fabsf(y * x - 1.0f);
        worst = fmaxf(worst, err);
    }
    out[2] = worst;
}
int main() {
    float *d, h[3];
    cudaMalloc(&d, sizeof(h));
    k<<<1, 1>>>(d, 1.0f, -0.0f);
    cudaMemcpy(h, d, sizeof(h), cudaMemcpyDeviceToHost);
    unsigned u0, u1;
    memcpy(&u0, &h[0], 4); memcpy(&u1, &h[1], 4);
    printf("rcp.approx(1) = %.9g (0x%08x)  ex2.approx(-0) = %.9g (0x%08x)  max |x rcp(x) - 1| on [1,2) = %.3g\n", h[0], u0, h[1], u1, h[2]);
    return (u0 == 0x3f800000u && u1 == 0x3f800000u) ? 0 : 1;
}
