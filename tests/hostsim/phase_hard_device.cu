/*
 * tests/hostsim/phase_hard_device.cu — TEST-ONLY: the device functions of the phase pass and the K2 walk on chosen
 * samples, for tests/test_gpu_phase_hard.py.  Built at test time with the library's nvcc and flags.
 *
 * k2a_phase_mag_warps and the K2 walk evaluate vdl2_phase_fast_nb, vdl2_mag_fast, vdl2_mag_fast_nb, vdl2_phase_of and
 * vdl2_mag_of on samples no public call lets a caller choose one by one; phase_hard_run evaluates each of them on n
 * samples and returns per sample
 *   val[i][0..3]  vdl2_phase_fast, vdl2_phase_fast_nb, vdl2_mag_fast, vdl2_mag_fast_nb (the fast float)
 *   val[i][4..5]  vdl2_phase_of, vdl2_mag_of (the fall-backs, and what the tail rows of the phase pass use)
 *   val[i][6]     (float) of libdevice's double atan2: what vdl2_phase_of returned before it took vdl2_atan2_cr
 *   slow[i][0..3] the *slow flags of the four fast routines
 */
#include <cuda_runtime.h>
#include "vdl2_core.cuh"

__constant__ double c_phase_hard_tab[VDL2_ATAN_TABLE_DOUBLES] = VDL2_ATAN_TABLE_INIT;

__global__ void phase_hard_kernel(const float2 *x, int n, float *val, int *slow) {
	__shared__ double s_tab[VDL2_ATAN_TABLE_DOUBLES];
	if(threadIdx.x < VDL2_ATAN_TABLE_DOUBLES) s_tab[threadIdx.x] = c_phase_hard_tab[threadIdx.x];
	__syncthreads();
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if(i >= n) return;
	const float2 d = x[i];
	float *v = val + 7 * (size_t)i;
	int *s = slow + 4 * (size_t)i;
	v[0] = vdl2_phase_fast(d.x, d.y, s_tab, &s[0]);
	v[1] = vdl2_phase_fast_nb(d.x, d.y, s_tab, &s[1]);
	v[2] = vdl2_mag_fast(d.x, d.y, &s[2]);
	v[3] = vdl2_mag_fast_nb(d.x, d.y, &s[3]);
	v[4] = vdl2_phase_of(d.x, d.y);
	v[5] = vdl2_mag_of(d.x, d.y);
	v[6] = __double2float_rn(atan2((double)d.y, (double)d.x));
}

extern "C" int phase_hard_run(const float *x, int n, float *val, int *slow) {
	float2 *dx = nullptr;
	float *dv = nullptr;
	int *ds = nullptr;
	int rc = 1;
	if(cudaMalloc(&dx, sizeof(float2) * n) == cudaSuccess && cudaMalloc(&dv, sizeof(float) * 7 * n) == cudaSuccess &&
	   cudaMalloc(&ds, sizeof(int) * 4 * n) == cudaSuccess &&
	   cudaMemcpy(dx, x, sizeof(float2) * n, cudaMemcpyHostToDevice) == cudaSuccess) {
		phase_hard_kernel<<<(n + 127) / 128, 128>>>(dx, n, dv, ds);
		if(cudaGetLastError() == cudaSuccess && cudaDeviceSynchronize() == cudaSuccess &&
		   cudaMemcpy(val, dv, sizeof(float) * 7 * n, cudaMemcpyDeviceToHost) == cudaSuccess &&
		   cudaMemcpy(slow, ds, sizeof(int) * 4 * n, cudaMemcpyDeviceToHost) == cudaSuccess)
			rc = 0;
	}
	cudaFree(dx); cudaFree(dv); cudaFree(ds);
	return rc;
}
