// Multi-GPU gather (NCCL) and the JPEG decode front-end (nvJPEG), both loaded at run time (C ABI: include/pf_b200.h).
#include <cstring>

#include "host.h"
#include "comm.cuh"
#include "jpeg.cuh"

using namespace pf;

extern "C" {

// ---- multi-GPU gather (NCCL point-to-point; SURVEY.md 8e) ---------------------------------------------------
#define NCCL_TRY(expr)                                                                                              \
  do {                                                                                                              \
    int r__ = (expr);                                                                                               \
    if (r__ != kNcclSuccess) return fail(PF_ERR_CUDA, "%s: %s", #expr, api.GetErrorString ? api.GetErrorString(r__) : "NCCL error"); \
  } while (0)
int pf_comm_unique_id(void* id128) {
  if (!id128) return fail(PF_ERR_ARG, "pf_comm_unique_id: null argument");
  const NcclApi& api = nccl_api();
  if (api.error) return fail(PF_ERR_CUDA, "%s", api.error);
  static_assert(sizeof(NcclUniqueId) == 128, "ncclUniqueId is 128 bytes");
  NCCL_TRY(api.GetUniqueId((NcclUniqueId*)id128));
  return PF_OK;
}
int pf_comm_create(int device, int rank, int nranks, const void* id128, pf_comm_handle* out) {
  if (!id128 || !out || nranks < 1 || rank < 0 || rank >= nranks) return fail(PF_ERR_ARG, "pf_comm_create: bad argument");
  const NcclApi& api = nccl_api();
  if (api.error) return fail(PF_ERR_CUDA, "%s", api.error);
  CU(cudaSetDevice(device));
  NcclUniqueId id;
  memcpy(&id, id128, sizeof id);
  pf_comm* c = new pf_comm();
  c->device = device; c->rank = rank; c->nranks = nranks;
  const int r = api.CommInitRank(&c->comm, nranks, id, rank);
  if (r != kNcclSuccess) { delete c; return fail(PF_ERR_CUDA, "ncclCommInitRank: %s", api.GetErrorString(r)); }
  *out = c;
  return PF_OK;
}
int pf_comm_destroy(pf_comm_handle c) {
  if (!c) return PF_OK;
  const NcclApi& api = nccl_api();
  cudaSetDevice(c->device);
  if (c->comm && api.CommDestroy) api.CommDestroy(c->comm);
  delete c;
  return PF_OK;
}
int pf_gather(pf_comm_handle c, int root, int count, void* const* dev_ptrs, const int64_t* bytes, const int32_t* peer, void* stream) {
  if (!c || count < 0 || root < 0 || root >= c->nranks || (count > 0 && (!dev_ptrs || !bytes))) return fail(PF_ERR_ARG, "pf_gather: bad argument");
  if (c->rank == root && count > 0 && !peer) return fail(PF_ERR_ARG, "pf_gather: the root needs the source rank of every segment");
  const NcclApi& api = nccl_api();
  CU(cudaSetDevice(c->device));
  if (count == 0) return PF_OK;
  NCCL_TRY(api.GroupStart());
  for (int i = 0; i < count; ++i) {
    int r;
    if (c->rank == root) {
      if (peer[i] < 0 || peer[i] >= c->nranks || peer[i] == root) { api.GroupEnd(); return fail(PF_ERR_ARG, "pf_gather: segment %d comes from rank %d", i, peer[i]); }
      r = api.Recv(dev_ptrs[i], (size_t)bytes[i], kNcclUint8, peer[i], c->comm, (cudaStream_t)stream);
    } else {
      r = api.Send(dev_ptrs[i], (size_t)bytes[i], kNcclUint8, root, c->comm, (cudaStream_t)stream);
    }
    if (r != kNcclSuccess) { api.GroupEnd(); return fail(PF_ERR_CUDA, "ncclSend/Recv: %s", api.GetErrorString(r)); }
  }
  NCCL_TRY(api.GroupEnd());
  return PF_OK;
}

// ---- decode front-end (nvJPEG; SURVEY.md 8f-2) ------------------------------------------------------------------
int pf_jpeg_create(int device, int max_threads, pf_jpeg_handle* out) {
  if (!out) return fail(PF_ERR_ARG, "pf_jpeg_create: null argument");
  const NvjpegApi& api = nvjpeg_api();
  if (api.error) return fail(PF_ERR_CUDA, "%s", api.error);
  CU(cudaSetDevice(device));
  pf_jpeg* j = new pf_jpeg();
  j->device = device;
  if (api.CreateSimple(&j->handle) != NVJPEG_STATUS_SUCCESS) { delete j; return fail(PF_ERR_CUDA, "nvjpegCreateSimple failed"); }
  int nt = max_threads > 0 ? max_threads : (int)std::thread::hardware_concurrency() / 2;
  nt = nt < 1 ? 1 : (nt > 32 ? 32 : nt);
  j->workers.resize(nt);
  bool ok = cudaEventCreateWithFlags(&j->start, cudaEventDisableTiming) == cudaSuccess;
  for (auto& w : j->workers) {
    ok = ok && api.StateCreate(j->handle, &w.state) == NVJPEG_STATUS_SUCCESS;
    ok = ok && cudaStreamCreateWithFlags(&w.stream, cudaStreamNonBlocking) == cudaSuccess;
    ok = ok && cudaEventCreateWithFlags(&w.done, cudaEventDisableTiming) == cudaSuccess;
  }
  if (!ok) { pf_jpeg_destroy(j); return fail(PF_ERR_CUDA, "pf_jpeg_create: decoder state / stream creation failed"); }
  *out = j;
  return PF_OK;
}
int pf_jpeg_destroy(pf_jpeg_handle j) {
  if (!j) return PF_OK;
  const NvjpegApi& api = nvjpeg_api();
  cudaSetDevice(j->device);
  for (auto& w : j->workers) {
    if (w.stream) cudaStreamSynchronize(w.stream);
    if (w.state) api.StateDestroy(w.state);
    if (w.stream) cudaStreamDestroy(w.stream);
    if (w.done) cudaEventDestroy(w.done);
  }
  if (j->start) cudaEventDestroy(j->start);
  if (j->handle) api.Destroy(j->handle);
  delete j;
  return PF_OK;
}
int pf_jpeg_info(pf_jpeg_handle j, const uint8_t* data, int64_t length, int32_t* height, int32_t* width) {
  if (!j || !data || length < 4 || !height || !width) return fail(PF_ERR_ARG, "pf_jpeg_info: bad argument");
  const NvjpegApi& api = nvjpeg_api();
  int nc = 0, ws[NVJPEG_MAX_COMPONENT] = {0}, hs[NVJPEG_MAX_COMPONENT] = {0};
  nvjpegChromaSubsampling_t ss;
  if (api.GetImageInfo(j->handle, data, (size_t)length, &nc, &ss, ws, hs) != NVJPEG_STATUS_SUCCESS) return fail(PF_ERR_ARG, "pf_jpeg_info: not a decodable JPEG stream");
  *height = hs[0]; *width = ws[0];
  return PF_OK;
}
int pf_jpeg_decode_batch(pf_jpeg_handle j, int n, const uint8_t* const* data, const int64_t* length, const int32_t* height, const int32_t* width,
                         uint8_t* blob, const int64_t* offset, void* stream) {
  if (!j || n < 1 || !data || !length || !height || !width || !blob || !offset) return fail(PF_ERR_ARG, "pf_jpeg_decode_batch: bad argument");
  const NvjpegApi& api = nvjpeg_api();
  CU(cudaSetDevice(j->device));
  cudaStream_t st = (cudaStream_t)stream;
  // the workers' streams start after everything already queued on the caller's stream (the blob may be in use by an earlier forward)
  CU(cudaEventRecord(j->start, st));
  const int nt = (int)j->workers.size() < n ? (int)j->workers.size() : n;
  std::atomic<int> next{0}, failed{-1};
  auto work = [&](int t) {
    cudaSetDevice(j->device);
    pf_jpeg::Worker& w = j->workers[t];
    cudaStreamWaitEvent(w.stream, j->start, 0);
    for (int i = next.fetch_add(1); i < n; i = next.fetch_add(1)) {
      nvjpegImage_t dst{};
      dst.channel[0] = blob + offset[i];
      dst.pitch[0] = (size_t)width[i] * 3;
      if (api.Decode(j->handle, w.state, data[i], (size_t)length[i], NVJPEG_OUTPUT_BGRI, &dst, w.stream) != NVJPEG_STATUS_SUCCESS) failed.store(i);
    }
    cudaEventRecord(w.done, w.stream);
  };
  std::vector<std::thread> threads;
  for (int t = 1; t < nt; ++t) threads.emplace_back(work, t);
  work(0);
  for (auto& th : threads) th.join();
  for (int t = 0; t < nt; ++t) CU(cudaStreamWaitEvent(st, j->workers[t].done, 0));
  if (failed.load() >= 0) return fail(PF_ERR_ARG, "pf_jpeg_decode_batch: image %d could not be decoded", failed.load());
  return PF_OK;
}

}  // extern "C"
