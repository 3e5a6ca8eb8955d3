// Micro-benchmark: issue rates of the integer instructions the scan kernel is made of, alone and mixed (developer tool).
// nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o pipes pipes.cu && ./pipes
#include <cstdio>
#include <cuda_runtime.h>
#define ITERS 4096
template <int MODE>
__global__ void k(unsigned* out, unsigned m1, unsigned m2, unsigned sh) {
  unsigned a = threadIdx.x * 2654435761u + m1, b = a ^ m2, c = a + 12345u, d = b * 3u + 1u;
  unsigned e = a ^ 0x9e3779b9u, f = b + 77u, g = c ^ 0x1234567u, h = d + 999u;
#pragma unroll 1
  for (int i = 0; i < ITERS; ++i) {
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (MODE == 0) { a = (a & m1) ^ b; b = (b | m2) ^ c; c = (c & m1) ^ d; d = (d | m2) ^ a; e = (e & m1) ^ f; f = (f | m2) ^ g; g = (g & m1) ^ h; h = (h | m2) ^ e; }          // LOP3 x8
      if (MODE == 1) { a = (a >> 1) ; b = __funnelshift_r(b, a, 3); c = c >> 2; d = __funnelshift_r(d, c, 5); e = e >> 1; f = __funnelshift_r(f, e, 3); g = g >> 2; h = __funnelshift_r(h, g, 5);
                       a ^= m1; c ^= m2; e ^= m1; g ^= m2; }   // SHF x8 + LOP x4
      if (MODE == 2) { a = a * m1 + b; b = b * m2 + c; c = c * m1 + d; d = d * m2 + a; e = e * m1 + f; f = f * m2 + g; g = g * m1 + h; h = h * m2 + e; }                            // IMAD x8
      if (MODE == 3) { a = __umulhi(a, m1) ^ b; b = __umulhi(b, m2) ^ c; c = __umulhi(c, m1) ^ d; d = __umulhi(d, m2) ^ a; e = __umulhi(e, m1) ^ f; f = __umulhi(f, m2) ^ g; g = __umulhi(g, m1) ^ h; h = __umulhi(h, m2) ^ e; }  // IMAD.HI x8 + LOP x8
      if (MODE == 4) { a = (a & m1) ^ b; b = b * m2 + c; c = (c & m1) ^ d; d = d * m2 + a; e = (e & m1) ^ f; f = f * m2 + g; g = (g & m1) ^ h; h = h * m2 + e; }                    // LOP3 x4 + IMAD x4
      if (MODE == 5) { a = (a & m1) ^ b; b = (b >> 1) ^ c; c = (c & m1) ^ d; d = (d >> 3) ^ a; e = (e & m1) ^ f; f = (f >> 1) ^ g; g = (g & m1) ^ h; h = (h >> 3) ^ e; }            // LOP3 x8 + SHF x4
      if (MODE == 6) { a = (a & m1) ^ b; b = __umulhi(b, m2) ^ c; c = (c & m1) ^ d; d = __umulhi(d, m2) ^ a; e = (e & m1) ^ f; f = __umulhi(f, m2) ^ g; g = (g & m1) ^ h; h = __umulhi(h, m2) ^ e; }  // LOP3 x8 + IMAD.HI x4
      if (MODE == 7) { a = (a & m1) ^ b; b = (b * sh) ^ c; c = (c & m1) ^ d; d = (d * sh) ^ a; e = (e & m1) ^ f; f = (f * sh) ^ g; g = (g & m1) ^ h; h = (h * sh) ^ e; }            // LOP3 x8 + IMAD x4
      if (MODE == 8) { a = __popc(a) + b; b = __popc(b) + c; c = __popc(c) + d; d = __popc(d) + a; e = __popc(e) + f; f = __popc(f) + g; g = __popc(g) + h; h = __popc(h) + e; }    // POPC x8 + IADD x8
      if (MODE == 9) { a = __byte_perm(a, b, m1); b = __byte_perm(b, c, m2); c = __byte_perm(c, d, m1); d = __byte_perm(d, a, m2); e = __byte_perm(e, f, m1); f = __byte_perm(f, g, m2); g = __byte_perm(g, h, m1); h = __byte_perm(h, e, m2); }  // PRMT x8
    }
  }
  out[blockIdx.x * blockDim.x + threadIdx.x] = a ^ b ^ c ^ d ^ e ^ f ^ g ^ h;
}
template <int MODE>
void run(const char* name, int ops) {
  int sms, khz; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0); cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
  unsigned* out; cudaMalloc(&out, sms * 8 * 256 * 4);
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  k<MODE><<<sms * 8, 256>>>(out, 0x55555555u, 0x33333333u, 4u);
  cudaEventRecord(e0);
  k<MODE><<<sms * 8, 256>>>(out, 0x55555555u, 0x33333333u, 4u);
  cudaEventRecord(e1); cudaEventSynchronize(e1);
  float ms; cudaEventElapsedTime(&ms, e0, e1);
  double warp_instr = (double)sms * 8 * 8 * ITERS * 4 * ops;      // per kernel
  double cyc = ms * 1e-3 * khz * 1e3;                              // at the maximum SM clock the device reports
  printf("%-28s %7.3f ms  %6.2f warp-instr/clk/SM (of the %d counted ops per group)\n", name, ms, warp_instr / cyc / sms, ops);
  cudaFree(out);
}
int main() {
  run<0>("LOP3 x8", 8); run<1>("SHF x8 + LOP x4", 12); run<2>("IMAD x8", 8); run<3>("IMAD.HI x8 + LOP x8", 16);
  run<4>("LOP3 x4 + IMAD x4", 8); run<5>("LOP3 x8 + SHF x4", 12); run<6>("LOP3 x8 + IMAD.HI x4", 12); run<7>("LOP3 x8 + IMAD x4", 12);
  run<8>("POPC x8 + IADD x8", 16); run<9>("PRMT x8", 8);
  return 0;
}
