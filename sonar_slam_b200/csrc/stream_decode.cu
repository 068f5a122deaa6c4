// Host side shared by the compressed-stream decoders (stream_decode.cuh).
#include <algorithm>

#include "stream_decode.cuh"

namespace sfe {

bool offsets_ok(const int64_t *offsets, int n) {
  for (int i = 0; i < n; ++i)
    if (offsets[i + 1] < offsets[i] || offsets[i] < 0) return false;
  return true;
}

ChunkStager::~ChunkStager() {
  if (copy) cudaStreamSynchronize(copy), cudaStreamDestroy(copy);
  for (int k = 0; k < 2; ++k) {
    if (ev_copied[k]) cudaEventDestroy(ev_copied[k]);
    if (ev_used[k]) cudaEventDestroy(ev_used[k]);
    if (pin[k]) cudaFreeHost(pin[k]);
    if (dev[k].ptr) cudaFree(dev[k].ptr);
  }
  if (ev_ready) cudaEventDestroy(ev_ready);
}

int ChunkStager::reserve(sfe_ctx *ctx, size_t in_max) {
  if (!copy) {
    SFE_CUDA(cudaStreamCreateWithFlags(&copy, cudaStreamNonBlocking));
    for (int k = 0; k < 2; ++k) {
      SFE_CUDA(cudaEventCreateWithFlags(&ev_copied[k], cudaEventDisableTiming));
      SFE_CUDA(cudaEventCreateWithFlags(&ev_used[k], cudaEventDisableTiming));
    }
    SFE_CUDA(cudaEventCreateWithFlags(&ev_ready, cudaEventDisableTiming));
  }
  SFE_CUDA(cudaStreamSynchronize(copy));
  for (int k = 0; k < 2; ++k) {
    int rc = ensure(ctx, dev[k], in_max);
    if (rc != SFE_OK) return rc;
    if (pin_cap[k] < in_max) {
      if (pin[k]) SFE_CUDA(cudaFreeHost(pin[k]));
      pin[k] = nullptr, pin_cap[k] = 0;
      SFE_CUDA(cudaMallocHost((void **)&pin[k], in_max + in_max / 4));
      pin_cap[k] = in_max + in_max / 4;
    }
  }
  SFE_CUDA(cudaEventRecord(ev_ready, ctx->stream));
  SFE_CUDA(cudaStreamWaitEvent(copy, ev_ready, 0));
  return SFE_OK;
}

int ChunkStager::acquire(uint8_t **pin_block) {
  turn ^= 1;
  SFE_CUDA(cudaEventSynchronize(ev_copied[turn]));
  *pin_block = pin[turn];
  return SFE_OK;
}

int ChunkStager::upload(sfe_ctx *ctx, size_t bytes, uint8_t **dev_block) {
  uint8_t *d = static_cast<uint8_t *>(dev[turn].ptr);
  SFE_CUDA(cudaStreamWaitEvent(copy, ev_used[turn], 0));  // the kernels of two chunks ago are done with it
  SFE_CUDA(cudaMemcpyAsync(d, pin[turn], bytes, cudaMemcpyHostToDevice, copy));
  SFE_CUDA(cudaEventRecord(ev_copied[turn], copy));
  SFE_CUDA(cudaStreamWaitEvent(ctx->stream, ev_copied[turn], 0));
  *dev_block = d;
  return SFE_OK;
}

int ChunkStager::done(sfe_ctx *ctx) {
  SFE_CUDA(cudaEventRecord(ev_used[turn], ctx->stream));
  return SFE_OK;
}

StreamDecoder::~StreamDecoder() {
  for (Buffer *b : {&status, &out})
    if (b->ptr) cudaFree(b->ptr);
}

int StreamDecoder::reserve_common(sfe_ctx *ctx, int n, size_t in_max, size_t out_bytes) {
  int rc = ensure(ctx, status, 4 * (size_t)n + 16);
  if (rc == SFE_OK && out_bytes) rc = ensure(ctx, out, out_bytes);
  return rc == SFE_OK ? stager.reserve(ctx, in_max) : rc;
}

int decode_all(sfe_ctx *ctx, StreamDecoder *(*decoder)(sfe_ctx *), const uint8_t *bytes, const int64_t *offsets, int n,
               int R, int B, uint8_t *out_dev, uint8_t *out_host, int32_t *status_host, const char *what) {
  SFE_REQUIRE(ctx && bytes && offsets && status_host, "%s: null argument", what);
  SFE_REQUIRE(n >= 0 && R > 0 && B > 0, "%s: bad shape n=%d R=%d B=%d", what, n, R, B);
  SFE_REQUIRE(offsets_ok(offsets, n), "%s: offsets must be non-decreasing", what);
  if (n == 0) return SFE_OK;
  SFE_CUDA(cudaSetDevice(ctx->device));
  StreamDecoder *dec = decoder(ctx);
  dec->parse(bytes, offsets, n, R, B, nullptr);
  const size_t fb = (size_t)R * B;
  const int chunk = dec->chunk_frames(ctx);
  const bool via_out = !out_dev;
  int rc = dec->reserve(ctx, chunk, via_out ? fb * chunk : 0);
  for (int f0 = 0; rc == SFE_OK && f0 < n; f0 += chunk) {
    const int nf = std::min(chunk, n - f0);
    uint8_t *o = via_out ? static_cast<uint8_t *>(dec->out.ptr) : out_dev + fb * f0;
    rc = dec->decode_chunk(ctx, f0, nf, o);
    if (rc == SFE_OK && out_host) {
      cudaError_t e = cudaMemcpyAsync(out_host + fb * f0, o, fb * nf, cudaMemcpyDeviceToHost, ctx->stream);
      if (e != cudaSuccess) rc = SFE_ERR_CUDA, set_error("%s: %s", what, cudaGetErrorString(e));
    }
  }
  if (rc != SFE_OK) return rc;
  SFE_CUDA(cudaMemcpyAsync(status_host, dec->status.ptr, 4 * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  SFE_CUDA(cudaStreamSynchronize(ctx->stream));
  return SFE_OK;
}

}  // namespace sfe
