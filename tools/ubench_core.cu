// Micro-benchmark: what issue rate can the smoothing kernel's arithmetic reach on sm_90a?
// One CTA of 512 threads per SM (4 warps per sub-partition, like qs_smooth_kernel), bodies that
// look like its inner loops.  Prints warp-instructions per clock per sub-partition.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -fmad=false -o ubench_core ubench_core.cu
#include <cstdio>
#include <cuda_runtime.h>

__device__ __forceinline__ float mul1(float a, float b) { float r; asm volatile("mul.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r; }
__device__ __forceinline__ float add1(float a, float b) { float r; asm volatile("add.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r; }
__device__ __forceinline__ float sat1(float a, float b) { float r; asm volatile("add.rn.sat.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(-fabsf(b))); return r; }
__device__ __forceinline__ unsigned prmt(unsigned a, unsigned s) { unsigned r; asm volatile("prmt.b32 %0, %1, 0x3F800000, %2;" : "=r"(r) : "r"(a), "r"(s)); return r; }

// MODE 0 FMUL, 1 FADD, 2 FADD.SAT, 3 CORE mix from registers, 4 CORE mix + LDS.128 weights,
// 5 = 4 + 8 PRMT per 7x4 terms, 6 = CORE with the clamp as FADD + FMNMX (ALU pipe)
template <int MODE> __global__ void __launch_bounds__(512, 1) k(float *out, int iters, float seed, long long *cyc) {
	__shared__ float tab[1024];
	for (int i = threadIdx.x; i < 1024; i += blockDim.x) tab[i] = 1.0f + i * 1e-6f;
	__syncthreads();
	float a2[4], a3[4], d[8], R[4], w[8];
	unsigned px = threadIdx.x * 0x01010101u;
	for (int i = 0; i < 4; i++) { a2[i] = seed; a3[i] = seed * 2; R[i] = 0.5f + i * 0.01f; }
	for (int i = 0; i < 8; i++) { d[i] = (threadIdx.x + i) * 1e-4f; w[i] = 1.0f + i * 1e-3f; }
	long long t0 = clock64();
	for (int it = 0; it < iters; it++) {
		if (MODE <= 2) {
#pragma unroll
			for (int r = 0; r < 28; r++)
#pragma unroll
				for (int i = 0; i < 8; i++) d[i] = MODE == 0 ? mul1(d[i], w[i]) : MODE == 1 ? add1(d[i], w[i]) : sat1(w[i], d[i]);
		} else {
			const float *tp = tab + (it & 7) * 32;
#pragma unroll
			for (int c = 0; c < 4; c++) {
				if (MODE >= 4) {
					float4 wa = *(const float4 *)(tp + c * 8), wb = *(const float4 *)(tp + c * 8 + 4);
					w[0] = wa.x; w[1] = wa.y; w[2] = wa.z; w[3] = wa.w; w[4] = wb.x; w[5] = wb.y; w[6] = wb.z; w[7] = wb.w;
				}
#pragma unroll
				for (int x = 0; x < 7; x++) {
					float t;
					if (MODE == 6) { t = add1(R[c], -fabsf(d[x])); t = fmaxf(t, 0.0f); }
					else t = sat1(R[c], d[x]);
					t = mul1(t, t);
					float a0 = mul1(d[x], t), a1 = mul1(w[x], t);
					a2[c] = add1(a2[c], mul1(a0, a1)); a3[c] = add1(a3[c], mul1(a1, a1));
				}
				if (MODE == 5) { d[2 * c] = __uint_as_float(prmt(px, 0x7604 + 16 * c)); d[2 * c + 1] = __uint_as_float(prmt(px, 0x7614 + 16 * c)); px += 0x01010101u; }
			}
		}
	}
	long long t1 = clock64();
	float s = 0;
	for (int i = 0; i < 4; i++) s += a2[i] + a3[i];
	for (int i = 0; i < 8; i++) s += d[i];
	out[blockIdx.x * blockDim.x + threadIdx.x] = s;
	if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}

template <int MODE> static void run(const char *name, double inst_per_iter) {
	int dev = 0, nsm = 0;
	cudaGetDevice(&dev);
	cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev);     /* one CTA per SM */
	float *out; long long *cyc, *h = new long long[nsm];
	cudaMalloc(&out, (size_t)nsm * 512 * 4); cudaMalloc(&cyc, (size_t)nsm * 8);
	int iters = 20000;
	k<MODE><<<nsm, 512>>>(out, 100, 1.0f, cyc);
	k<MODE><<<nsm, 512>>>(out, iters, 1.0f, cyc);
	cudaMemcpy(h, cyc, (size_t)nsm * 8, cudaMemcpyDeviceToHost);
	double c = 0; for (int i = 0; i < nsm; i++) c += h[i];
	c /= nsm;
	delete[] h;
	// 16 warps per SM, 4 per sub-partition: warp-instructions per sub-partition = 4 * per-warp count
	printf("%-44s %7.0f cycles  %.3f warp-instr/clk/sub-partition (counted FP%s instructions only)\n", name, c,
			4.0 * inst_per_iter * iters / c, MODE >= 5 ? "+PRMT" : "");
	cudaFree(out); cudaFree(cyc);
}

int main() {
	run<0>("FMUL stream (ILP 8)", 28 * 8);
	run<1>("FADD stream (ILP 8)", 28 * 8);
	run<2>("FADD.SAT -|x| stream (ILP 8)", 28 * 8);
	run<3>("CORE mix, weights in registers", 4 * 7 * 8);
	run<4>("CORE mix + 2 LDS.128 per coefficient", 4 * 7 * 8);
	run<5>("CORE mix + LDS + 2 PRMT per coefficient", 4 * 7 * 8 + 8);
	run<6>("CORE with FADD + FMNMX clamp (9 per term)", 4 * 7 * 9);
	return 0;
}
