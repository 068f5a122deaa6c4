// Host side shared by the compressed-stream decoders (jpeg.cu, png.cu) and the front end that feeds on them
// (pipeline.cu): the chunked upload of the streams' bytes, the batch of parsed headers, the decoder interface and the
// whole-call driver of the sfe_<codec>_decode_* entry points.
#pragma once
#include <vector>

#include "common.cuh"
#include "stage_timer.cuh"

namespace sfe {

// offsets[0..n] of n packed streams: non-negative and non-decreasing
bool offsets_ok(const int64_t *offsets, int n);

// The bytes of a chunk of frames go to the device on a copy stream of their own, through two pinned blocks and two
// device blocks used in turn: the host fills the block of chunk k + 1 while chunk k copies or decodes.  A block is
// filled again (chunk k + 2) once its copy has landed (ev_copied) and the kernels of chunk k are done with its device
// copy (ev_used).
struct ChunkStager {
  cudaStream_t copy = nullptr;  // created on first use
  cudaEvent_t ev_copied[2] = {}, ev_used[2] = {}, ev_ready = nullptr;
  uint8_t *pin[2] = {};
  size_t pin_cap[2] = {};
  Buffer dev[2];
  int turn = 0;

  ChunkStager() = default;
  ChunkStager(const ChunkStager &) = delete;
  ChunkStager &operator=(const ChunkStager &) = delete;
  ~ChunkStager();
  // Both turns take in_max bytes.  Called before any work of the call is enqueued (the blocks are not reallocated
  // while the copy stream may use them); the copy stream is ordered after everything on ctx->stream so far.
  int reserve(sfe_ctx *ctx, size_t in_max);
  // upload, step 1: the next turn's pinned block, for the host to fill, once its previous copy has landed
  int acquire(uint8_t **pin_block);
  // upload, step 2: its first `bytes` bytes to the turn's device block, which ctx->stream waits for
  int upload(sfe_ctx *ctx, size_t bytes, uint8_t **dev_block);
  // after the chunk's kernels on ctx->stream: the turn's device block may be overwritten from here on
  int done(sfe_ctx *ctx);
};

// The headers of a call's n packed streams.  bytes and offsets point into the caller's arrays: valid during the call.
template <class Header>
struct StreamBatch {
  const uint8_t *bytes = nullptr;
  const int64_t *offsets = nullptr;
  int n = 0, R = 0, B = 0;
  const int32_t *shape = nullptr;  // optional int32 [n][2]: frame i must be shape[2i] x shape[2i + 1] instead of R x B
  std::vector<Header> hdr;

  int R_of(int i) const { return shape ? shape[2 * i] : R; }
  int B_of(int i) const { return shape ? shape[2 * i + 1] : B; }

  // Header::status 0 is a stream the decoder takes; one whose frame is not R x B (or its own shape) gets size_status
  void parse(const uint8_t *bytes_, const int64_t *offsets_, int n_, int R_, int B_, const int32_t *shape_,
             void (*parse_header)(const uint8_t *, int64_t, Header &), int size_status) {
    bytes = bytes_, offsets = offsets_, n = n_, R = R_, B = B_, shape = shape_;
    hdr.resize(n);
    for (int i = 0; i < n; ++i) {
      parse_header(bytes + offsets[i], offsets[i + 1] - offsets[i], hdr[i]);
      if (hdr[i].status == 0 && (hdr[i].H != R_of(i) || hdr[i].W != B_of(i))) hdr[i].status = size_status;
    }
  }
};

// A compressed-stream decoder (jpeg.cu: JpegState, png.cu: PngState), one per context, created on first use.  A call
// parses its streams' headers, reserves every buffer for its chunk size, then decodes chunk after chunk on
// ctx->stream.
struct StreamDecoder {
  ChunkStager stager;
  StageTimer timer;
  Buffer status;  // device int32 [n]: per-frame status of the call's frames
  Buffer out;     // device uint8 [chunk][R][B]: decoded frames of one chunk, for callers without a device destination

  virtual ~StreamDecoder();
  virtual int chunk_frames(const sfe_ctx *ctx) const = 0;  // chunk size of the decode entry points
  // shape: null (every frame R x B) or int32 [n][2], each frame's own R x B (valid until the call's last decode_chunk)
  virtual void parse(const uint8_t *bytes, const int64_t *offsets, int n, int R, int B, const int32_t *shape) = 0;
  virtual int frame_status(int i) const = 0;  // after parse: 0 when the decoder takes frame i
  virtual const char *message(int status) const = 0;
  // after parse: every buffer sized for the largest chunk of `chunk` frames, and out_bytes of `out`; a decode_chunk of
  // any subset of consecutive frames of such a chunk fits too
  virtual int reserve(sfe_ctx *ctx, int chunk, size_t out_bytes) = 0;
  // frames [f0, f0 + nf) into out_dev (uint8 [nf][R][B], R x B = frame f0's shape: the frames of one decode_chunk share
  // it), their statuses into `status` at [f0, f0 + nf); asynchronous on ctx->stream, the bytes go in through the stager
  virtual int decode_chunk(sfe_ctx *ctx, int f0, int nf, uint8_t *out_dev) = 0;

 protected:
  // the last step of reserve() for n frames: the buffers every decoder has, then the stager
  int reserve_common(sfe_ctx *ctx, int n, size_t in_max, size_t out_bytes);
};

StreamDecoder *jpeg_decoder(sfe_ctx *ctx);
StreamDecoder *png_decoder(sfe_ctx *ctx);

// The body of the sfe_<codec>_decode_* entry points: frames into out_dev (device, [n][R][B]) or, through the
// decoder's `out`, into out_host (or nowhere); statuses into status_host.  Returns once both are there.
int decode_all(sfe_ctx *ctx, StreamDecoder *(*decoder)(sfe_ctx *), const uint8_t *bytes, const int64_t *offsets, int n,
               int R, int B, uint8_t *out_dev, uint8_t *out_host, int32_t *status_host, const char *what);

}  // namespace sfe
