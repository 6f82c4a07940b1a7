// gmap_intensity.h -- the C launchers of libtloam_b200_gmi.so (gmap_intensity.cu): the global map's intensity channel.
//
// libtloam_b200.so loads that library with dlopen on the first intensity call and resolves these symbols; nothing here
// defines a kernel, so including this header leaves the SASS of libtloam_b200.so alone.  Every pointer is a device pointer,
// every launch is enqueued on `stream` of `device`, and nothing synchronises.  The return value is a cudaError_t.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

// one frame of tloam_b200_global_map_append*_intensity, launched between k_gmap_emit and k_gmap_commit (the map's count is
// still the frame's base)
typedef struct tloam_gmi_frame {
  const double* reg;                          // [n x 3] registered scan (T.p), raw order
  const double* intensity;                    // [n] the raw scan's intensity, raw order
  unsigned n;
  const unsigned long long* minenc;           // [3] complemented min bound the voxel pipeline keyed the frame with
  double voxel;
  const unsigned long long* keys_sorted;      // [*n_vox] complemented voxel keys, descending (= ascending key)
  const unsigned* n_vox;                      // voxels of the frame
  const unsigned* refused;                    // the key-range guard refused the frame
  const unsigned long long* count;            // points in the map before this frame
  const unsigned long long* frames;           // frames in the map before this frame
  unsigned long long cap, frame_cap;          // the capacities k_gmap_emit / k_gmap_commit check
  double* map_intensity;                      // [cap] the intensity channel, parallel to the xyz map
  unsigned* state;                            // [2]: map has an intensity channel, a finite row found no voxel (sticky)
  int fresh;                                  // no intensity frame since the map was emptied: the map holds plain frames only
  void* scratch;                              // tloam_gmi_scratch_bytes(n) bytes
} tloam_gmi_frame;

size_t tloam_gmi_scratch_bytes(unsigned n);
// per-voxel average intensity of the frame at map_intensity[count + j] and the channel flag; *launches receives the count
int tloam_gmi_append(const tloam_gmi_frame* f, int device, cudaStream_t stream, int* launches);
// a frame appended without intensity: the map loses its channel if the frame adds any voxel
int tloam_gmi_plain(unsigned* state, const unsigned* n_vox, const unsigned* refused, const unsigned long long* count,
                    const unsigned long long* frames, unsigned long long cap, unsigned long long frame_cap, int device,
                    cudaStream_t stream);

typedef size_t (*tloam_gmi_scratch_bytes_fn)(unsigned);
typedef int (*tloam_gmi_append_fn)(const tloam_gmi_frame*, int, cudaStream_t, int*);
typedef int (*tloam_gmi_plain_fn)(unsigned*, const unsigned*, const unsigned*, const unsigned long long*, const unsigned long long*,
                                  unsigned long long, unsigned long long, int, cudaStream_t);

#ifdef __cplusplus
}
#endif
