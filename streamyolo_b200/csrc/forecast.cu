// Forecast of streaming detections (sAP/forecast/pps_forecast_kf.py): greedy IoU association of the tracks with each new
// detection, a batched constant-velocity Kalman filter, and the extrapolation of the tracks to a query frame.  One CTA per
// stream (sy_forecast_update, sy_forecast_extrap) or per sequence (sy_forecast_sequences); both run the same two device
// functions, forecast_update and forecast_extrap.  Compiled with -fmad=false: every fp32 / fp64 expression rounds each
// operation as the reference's numpy / torch CPU / pycocotools C code does, and the IoU spells its fp64 operations out.
#include "common.cuh"

namespace sy {

constexpr int kFcThreads = 256;
constexpr int kFcWarps = kFcThreads / 32;
constexpr int kFcMinSize = 75;               // extrap_clean_up's default min_size (forecast/__init__.py:33)

// per-stream scratch of forecast_update, in 4-byte words per track slot (see fc_scratch_words)
struct FcScratch {
  float* box;       // [T][4] the new detection's boxes, ltwh, in score order
  float* score;     // [T]
  int32_t* label;   // [T]
  int32_t* src;     // [T] new slot k: the matched track, or -1 for a new track
  int32_t* dsel;    // [T] new slot k: its detection (score order)
  int32_t* used;    // [T] track matched (match_fwd[i] is not None)
  float* x;         // [T][8] the new state, copied over the stream's state at the end
  float* P;         // [T][64]
  int32_t* nlabel;  // [T]
  float* nscore;    // [T]
  int32_t* ntrack;  // [T]
};
constexpr size_t kFcScratchWords = 4 + 1 + 1 + 1 + 1 + 1 + 8 + 64 + 1 + 1 + 1;

__device__ __forceinline__ FcScratch fc_scratch(void* ws, int s, int T) {
  uint32_t* w = reinterpret_cast<uint32_t*>(ws) + (size_t)s * T * kFcScratchWords;
  FcScratch q;
  q.box = reinterpret_cast<float*>(w);            w += (size_t)T * 4;
  q.score = reinterpret_cast<float*>(w);          w += T;
  q.label = reinterpret_cast<int32_t*>(w);        w += T;
  q.src = reinterpret_cast<int32_t*>(w);          w += T;
  q.dsel = reinterpret_cast<int32_t*>(w);         w += T;
  q.used = reinterpret_cast<int32_t*>(w);         w += T;
  q.x = reinterpret_cast<float*>(w);              w += (size_t)T * 8;
  q.P = reinterpret_cast<float*>(w);              w += (size_t)T * 64;
  q.nlabel = reinterpret_cast<int32_t*>(w);       w += T;
  q.nscore = reinterpret_cast<float*>(w);         w += T;
  q.ntrack = reinterpret_cast<int32_t*>(w);
  return q;
}

// one stream's (or sequence's) state inside SyForecastState
struct FcStream {
  float* x;         // [T][8]
  float* P;         // [T][64]
  int32_t* label;
  float* score;
  int32_t* track;
  int32_t* meta;    // [4] n_tracks, n_matched, next track id, overflow
};

__device__ __forceinline__ FcStream fc_stream(const SyForecastState& st, int s) {
  const size_t T = st.T;
  return FcStream{st.x + s * T * 8, st.P + s * T * 64, st.label + s * T, st.score + s * T, st.track + s * T,
                  st.meta + (size_t)s * 4};
}

// pycocotools' bbIou (maskApi.c) for one detection-track pair, iscrowd = 0: D = the track's box, G = the detection's,
// both ltwh widened to double.  Explicit _rn operations: no contraction may change a rounding.
__device__ __forceinline__ double bb_iou(const double D[4], const double G[4]) {
  const double da = __dmul_rn(D[2], D[3]), ga = __dmul_rn(G[2], G[3]);
  const double w = __dadd_rn(fmin(__dadd_rn(D[2], D[0]), __dadd_rn(G[2], G[0])), -fmax(D[0], G[0]));
  if (w <= 0) return 0.0;
  const double h = __dadd_rn(fmin(__dadd_rn(D[3], D[1]), __dadd_rn(G[3], G[1])), -fmax(D[1], G[1]));
  if (h <= 0) return 0.0;
  const double i = __dmul_rn(w, h);
  return __ddiv_rn(i, __dadd_rn(__dadd_rn(da, ga), -i));
}

// score order of np.argsort(scores)[::-1]: descending, NaN first (argsort puts NaN last), equal keys with the higher
// index first (a stable ascending sort, reversed)
__device__ __forceinline__ bool fc_before(float sk, int k, float sj, int j) {
  const bool nk = isnan(sk), nj = isnan(sj);
  if (nk != nj) return nk;
  if (nk || sk == sj) return k > j;
  return sk > sj;
}

// (iou, track) of a candidate beats (biou, bi): a higher IoU, or an equal one from a later track
__device__ __forceinline__ bool fc_better(double iou, int i, double biou, int bi) {
  return bi < 0 || iou > biou || (iou == biou && i > bi);
}

// Sum of 0 * v over the entries a matmul multiplies by F's zeros: 0 for finite values, NaN once one is not (0 * inf),
// which is how torch's F @ x spreads a non-finite component over the whole row.
__device__ __forceinline__ float zero_terms(const float* v, int stride, int skip0, int skip1) {
  float z = 0.f;
  for (int j = 0; j < 8; ++j)
    if (j != skip0 && j != skip1) z = z + 0.f * v[j * stride];
  return z;
}

// Kalman predict with F(dt) and Q = dt^2 I (pps_forecast_kf.py:64-79), in place: x = F x, P = F P F' + Q, with the
// matmuls' zero terms kept so that non-finite values spread as they do there.
__device__ __forceinline__ void kf_predict(float* x, float* P, float dt) {
  float xo[8];
  for (int r = 0; r < 8; ++r)
    xo[r] = (r < 4 ? x[r] + dt * x[r + 4] : x[r]) + zero_terms(x, 1, r, r < 4 ? r + 4 : r);
  for (int r = 0; r < 8; ++r) x[r] = xo[r];
  const float q = dt * dt;
  float fp[64];                                     // F P
  for (int r = 0; r < 8; ++r)
    for (int c = 0; c < 8; ++c)
      fp[r * 8 + c] = (r < 4 ? P[r * 8 + c] + dt * P[(r + 4) * 8 + c] : P[r * 8 + c]) +
                      zero_terms(P + c, 8, r, r < 4 ? r + 4 : r);
  for (int r = 0; r < 8; ++r)                       // (F P) F' + Q
    for (int c = 0; c < 8; ++c) {
      float v = (c < 4 ? fp[r * 8 + c] + dt * fp[r * 8 + c + 4] : fp[r * 8 + c]) +
                zero_terms(fp + r * 8, 1, c, c < 4 ? c + 4 : c);
      P[r * 8 + c] = v + (r == c ? q : 0.f);
    }
}

// Kalman update with H = [I 0], R = 10 I (batch_kf_update, :81-97): x += K (z - x[:4]), P -= K P[:4], K = P[:, :4] S^-1,
// S^-1 by Gauss-Jordan elimination with partial pivoting.  xo / Po may alias nothing of x / P.
__device__ __forceinline__ void kf_update(const float* x, const float* P, const float z[4], float* xo, float* Po) {
  float a[4][8];                                    // [S | I] -> [I | S^-1]
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 8; ++c) a[r][c] = c < 4 ? (r == c ? P[r * 8 + c] + 10.f : P[r * 8 + c]) : (c - 4 == r ? 1.f : 0.f);
  for (int k = 0; k < 4; ++k) {
    int p = k;
    for (int r = k + 1; r < 4; ++r)
      if (fabsf(a[r][k]) > fabsf(a[p][k])) p = r;
    if (p != k)
      for (int c = 0; c < 8; ++c) { const float t = a[k][c]; a[k][c] = a[p][c]; a[p][c] = t; }
    const float inv = __fdiv_rn(1.f, a[k][k]);
    for (int c = 0; c < 8; ++c) a[k][c] = a[k][c] * inv;
    for (int r = 0; r < 4; ++r) {
      if (r == k) continue;
      const float f = a[r][k];
      for (int c = 0; c < 8; ++c) a[r][c] = a[r][c] - f * a[k][c];
    }
  }
  float y[4];
  for (int r = 0; r < 4; ++r) y[r] = z[r] - x[r];
  for (int r = 0; r < 8; ++r) {
    float K[4];
    for (int c = 0; c < 4; ++c) {
      float s = 0.f;
      for (int k = 0; k < 4; ++k) s = s + P[r * 8 + k] * a[k][4 + c];
      K[c] = s;
    }
    float ky = 0.f;
    for (int c = 0; c < 4; ++c) ky = ky + K[c] * y[c];
    xo[r] = x[r] + ky;
    for (int c = 0; c < 8; ++c) {
      float s = 0.f;
      for (int k = 0; k < 4; ++k) s = s + K[k] * P[k * 8 + c];
      Po[r * 8 + c] = P[r * 8 + c] - s;
    }
  }
}

// One new detection for one stream (pps_forecast_kf.py:170-256 with --forecast-before-assoc and iou association), run by
// the whole CTA.  rows: sy_postprocess_nms rows [n][7] (x1, y1, x2, y2, obj, class_conf, class_pred); the score is
// obj * class_conf and the label (int)class_pred.  n > T leaves the state as it was and sets the overflow flag.
__device__ void forecast_update(const FcStream& S, const FcScratch& W, int T, const float* __restrict__ rows, int n,
                                int dt_i, bool start, double th, bool clear_on_empty) {
  __shared__ double s_iou[2][kFcWarps];
  __shared__ int s_idx[2][kFcWarps], s_last[2][kFcWarps], s_nan[2][kFcWarps];
  __shared__ int s_meta[3];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (n > T) {
    if (tid == 0) S.meta[3] = 1;
    return;
  }
  if (tid == 0) {
    if (start) S.meta[0] = S.meta[1] = S.meta[2] = 0;
    s_meta[0] = S.meta[0];
    s_meta[1] = S.meta[1];
    s_meta[2] = S.meta[2];
    S.meta[3] = 0;
  }
  __syncthreads();
  const int m = s_meta[0];
  int n_matched = s_meta[1], next_id = s_meta[2];
  const float dt = (float)dt_i;
  // predict every track before the association, on every new detection (:175-184)
  for (int i = tid; i < m; i += kFcThreads) kf_predict(S.x + (size_t)i * 8, S.P + (size_t)i * 64, dt);
  if (n == 0) {
    // pps_forecast_kf.py keeps the predicted tracks and n_matched; the streamer (sAP/forecast/streamer.py:247-280)
    // associates the tracks with nothing, matches none and starts from the empty detection: no track is left.  The
    // id counter stays either way.  (The predict above only wrote the tracks' own slots.)
    if (clear_on_empty && tid == 0) S.meta[0] = S.meta[1] = 0;
    return;
  }
  // sort by score (:204-207) by rank, convert ltrb -> ltwh (:209)
  for (int j = tid; j < n; j += kFcThreads) {
    const float* d = rows + (size_t)j * 7;
    const float sj = __fmul_rn(d[4], d[5]);
    int rank = 0;
    for (int k = 0; k < n; ++k) rank += fc_before(__fmul_rn(rows[(size_t)k * 7 + 4], rows[(size_t)k * 7 + 5]), k, sj, j);
    W.box[rank * 4 + 0] = d[0];
    W.box[rank * 4 + 1] = d[1];
    W.box[rank * 4 + 2] = __fsub_rn(d[2], d[0]);
    W.box[rank * 4 + 3] = __fsub_rn(d[3], d[1]);
    W.score[rank] = sj;
    W.label[rank] = (int)d[6];
  }
  for (int i = tid; i < m; i += kFcThreads) W.used[i] = 0;
  __syncthreads();
  // greedy association (track/__init__.py:90-133, no_unmatched1): detections in score order; each takes the unmatched
  // track of its label with the highest IoU >= th, a later track winning a tie.  The loop skips a track only when
  // `iou < best`, so a NaN IoU (a non-finite box) is taken and then every later eligible track replaces it: with a NaN
  // among the eligible tracks the last eligible track wins.  Every thread reduces the same warp winners, so all of them
  // hold the same decision; the owner of the track marks it used.
  int nm = 0;
  if (m > 0) {
    for (int j = 0; j < n; ++j) {
      const int lj = W.label[j];
      const double G[4] = {W.box[j * 4], W.box[j * 4 + 1], W.box[j * 4 + 2], W.box[j * 4 + 3]};
      double biou = 0.0;
      int bi = -1, last = -1, nan = 0;              // the last eligible track; a NaN IoU among the eligible ones
      for (int i = tid; i < m; i += kFcThreads) {
        if (W.used[i] || S.label[i] != lj) continue;
        const float* xi = S.x + (size_t)i * 8;
        const double D[4] = {xi[0], xi[1], xi[2], xi[3]};
        const double iou = bb_iou(D, G);
        last = i;
        nan |= isnan(iou);
        if (iou >= th && fc_better(iou, i, biou, bi)) biou = iou, bi = i;
      }
      for (int o = 16; o > 0; o >>= 1) {
        const double ov = __shfl_xor_sync(0xffffffffu, biou, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        last = max(last, __shfl_xor_sync(0xffffffffu, last, o));
        nan |= __shfl_xor_sync(0xffffffffu, nan, o);
        if (oi >= 0 && fc_better(ov, oi, biou, bi)) biou = ov, bi = oi;
      }
      const int par = j & 1;                        // two slots: one barrier per detection
      if (lane == 0) s_iou[par][warp] = biou, s_idx[par][warp] = bi, s_last[par][warp] = last, s_nan[par][warp] = nan;
      __syncthreads();
      biou = 0.0, bi = -1, last = -1, nan = 0;
      for (int w = 0; w < kFcWarps; ++w) {
        if (s_idx[par][w] >= 0 && fc_better(s_iou[par][w], s_idx[par][w], biou, bi)) biou = s_iou[par][w], bi = s_idx[par][w];
        last = max(last, s_last[par][w]);
        nan |= s_nan[par][w];
      }
      if (nan) bi = last;
      if (bi >= 0) {
        if (bi % kFcThreads == tid) W.used[bi] = 1;
        if (tid == 0) W.src[nm] = bi, W.dsel[nm] = j;
        ++nm;
      }
    }
    if (tid == 0) {                                 // order2 = matched2 + unmatched2
      int k = nm;
      for (int j = 0, q = 0; j < n; ++j) {
        if (q < nm && W.dsel[q] == j) { ++q; continue; }
        W.src[k] = -1, W.dsel[k] = j, ++k;
      }
    }
    next_id += n - nm;                              // iou_assoc's tkidx += n_unmatched2 (:131-132)
    __syncthreads();
  }
  if (nm > 0) {
    // matched tracks first, in match order, updated; then the unmatched detections as new tracks (:226-243)
    for (int k = tid; k < n; k += kFcThreads) {
      const int j = W.dsel[k], i = W.src[k];
      float* xo = W.x + (size_t)k * 8;
      float* Po = W.P + (size_t)k * 64;
      if (i >= 0) {
        const float z[4] = {W.box[j * 4], W.box[j * 4 + 1], W.box[j * 4 + 2], W.box[j * 4 + 3]};
        kf_update(S.x + (size_t)i * 8, S.P + (size_t)i * 64, z, xo, Po);
        W.ntrack[k] = S.track[i];
      } else {
        for (int c = 0; c < 8; ++c) xo[c] = c < 4 ? W.box[j * 4 + c] : 0.f;
        for (int c = 0; c < 64; ++c) Po[c] = (c % 9 == 0) ? 100.f : 0.f;
        W.ntrack[k] = next_id - (n - nm) + (k - nm);
      }
      W.nlabel[k] = W.label[j];
      W.nscore[k] = W.score[j];
    }
    n_matched = nm;
  } else {
    // no track matched, or none existed: start from the new detections (:245-253); the ids continue from the counter
    // iou_assoc advanced
    for (int k = tid; k < n; k += kFcThreads) {
      float* xo = W.x + (size_t)k * 8;
      float* Po = W.P + (size_t)k * 64;
      for (int c = 0; c < 8; ++c) xo[c] = c < 4 ? W.box[k * 4 + c] : 0.f;
      for (int c = 0; c < 64; ++c) Po[c] = (c % 9 == 0) ? 100.f : 0.f;
      W.nlabel[k] = W.label[k];
      W.nscore[k] = W.score[k];
      W.ntrack[k] = next_id + k;
    }
    next_id += n;
    if (m > 0) n_matched = 0;
  }
  __syncthreads();
  for (int e = tid; e < n * 8; e += kFcThreads) S.x[e] = W.x[e];
  for (int e = tid; e < n * 64; e += kFcThreads) S.P[e] = W.P[e];
  for (int k = tid; k < n; k += kFcThreads) {
    S.label[k] = W.nlabel[k];
    S.score[k] = W.nscore[k];
    S.track[k] = W.ntrack[k];
  }
  if (tid == 0) S.meta[0] = n, S.meta[1] = n_matched, S.meta[2] = next_id;
}

// The tracks extrapolated dt frames ahead (:258-273) and cleaned up as extrap_clean_up(..., lt=True) does
// (forecast/__init__.py:33-56), compacted in track order into box [.][4] (ltwh), score, label, track.  -> rows written.
// dt is an fp32 frame count: the streamer's fractional query (its Python float rounded to fp32 by numpy's fp32
// multiply), or an integer one converted exactly.
__device__ int forecast_extrap(const FcStream& S, float dt, float W_img, float H_img, float* __restrict__ box,
                               float* __restrict__ score, int32_t* __restrict__ label, int32_t* __restrict__ track) {
  __shared__ int s_cnt[kFcWarps];
  __shared__ int s_mt[2];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) s_mt[0] = S.meta[0], s_mt[1] = S.meta[1];
  __syncthreads();
  const int m = s_mt[0], n_matched = s_mt[1];
  int base = 0;
  for (int i0 = 0; i0 < m; i0 += kFcThreads) {
    const int i = i0 + tid;
    bool keep = false;
    float b[4];
    if (i < m) {
      const float* x = S.x + (size_t)i * 8;
      for (int c = 0; c < 4; ++c) b[c] = i < n_matched ? x[c] + dt * x[c + 4] : x[c];
      keep = b[2] > 0.f && b[3] > 0.f;
      float r = b[0] + b[2], btm = b[1] + b[3];
      // clip as np.clip does (NaN passes through)
      b[0] = b[0] < 0.f ? 0.f : (b[0] > W_img ? W_img : b[0]);
      r = r < 0.f ? 0.f : (r > W_img ? W_img : r);
      b[1] = b[1] < 0.f ? 0.f : (b[1] > H_img ? H_img : b[1]);
      btm = btm < 0.f ? 0.f : (btm > H_img ? H_img : btm);
      b[2] = r - b[0];
      b[3] = btm - b[1];
      keep = keep && (long long)b[2] * (long long)b[3] >= kFcMinSize;     // astype(int) truncates toward zero
    }
    const unsigned bal = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) s_cnt[warp] = __popc(bal);
    __syncthreads();
    int off = base, tot = 0;
    for (int w = 0; w < kFcWarps; ++w) {
      if (w < warp) off += s_cnt[w];
      tot += s_cnt[w];
    }
    if (keep) {
      const int o = off + __popc(bal & ((1u << lane) - 1u));
      for (int c = 0; c < 4; ++c) box[(size_t)o * 4 + c] = b[c];
      score[o] = S.score[i];
      label[o] = S.label[i];
      track[o] = S.track[i];
    }
    base += tot;
    __syncthreads();                                // s_cnt is rewritten by the next chunk
  }
  __syncthreads();                                  // and s_mt by the next call
  return base;
}

__global__ void __launch_bounds__(kFcThreads) forecast_update_kernel(const SyForecastUpdateDesc q) {
  const int s = blockIdx.x;
  if (q.keep != nullptr && q.keep[s] == 0) {        // no decoded frame: the stream is left untouched
    if (threadIdx.x == 0) q.state.meta[(size_t)s * 4 + 3] = 0;
    return;
  }
  const int n = min(max(q.count[s], 0), q.max_det);
  forecast_update(fc_stream(q.state, s), fc_scratch(q.workspace, s, q.state.T), q.state.T,
                  q.det + (size_t)s * q.max_det * 7, n, q.dt[s], q.start != nullptr && q.start[s] != 0, q.match_iou_th,
                  q.clear_on_empty != 0);
}

__global__ void __launch_bounds__(kFcThreads) forecast_extrap_kernel(const SyForecastExtrapDesc q) {
  const int s = blockIdx.x;
  const size_t T = q.state.T;
  const int n = forecast_extrap(fc_stream(q.state, s), (float)q.dt[s], (float)q.img_wh[s * 2],
                                (float)q.img_wh[s * 2 + 1], q.box_out + s * T * 4, q.score_out + s * T,
                                q.label_out + s * T, q.track_out + s * T);
  if (threadIdx.x == 0) q.count_out[s] = n;
}

// One CTA per (stream, query): blockIdx.x the stream, blockIdx.y the query; queries past n_query[s] write a count of 0.
__global__ void __launch_bounds__(kFcThreads) forecast_extrap_queries_kernel(const SyForecastExtrapQueriesDesc q) {
  const int s = blockIdx.x, k = blockIdx.y;
  const size_t T = q.state.T, o = (size_t)s * q.Q + k;
  if (k >= q.n_query[s]) {
    if (threadIdx.x == 0) q.count_out[o] = 0;
    return;
  }
  const int n = forecast_extrap(fc_stream(q.state, s), q.dt[o], (float)q.img_wh[s * 2], (float)q.img_wh[s * 2 + 1],
                                q.box_out + o * T * 4, q.score_out + o * T, q.label_out + o * T, q.track_out + o * T);
  if (threadIdx.x == 0) q.count_out[o] = n;
}

// One CTA per sequence: its annotated frames in order, each a table row (see SyForecastSequencesDesc).
__global__ void __launch_bounds__(kFcThreads) forecast_sequences_kernel(const SyForecastSequencesDesc q) {
  const int s = blockIdx.x;
  const FcStream S = fc_stream(q.state, s);
  const FcScratch W = fc_scratch(q.workspace, s, q.state.T);
  int prev = -1;
  bool start = true;
  for (int f = q.seq_frames[s]; f < q.seq_frames[s + 1]; ++f) {
    const int32_t* row = q.frames + (size_t)f * 6;
    const int d = row[0];
    if (d < 0) {                                    // no detection out yet: nothing emitted
      if (threadIdx.x == 0) q.rows_out[f] = 0;
      continue;
    }
    if (d != prev) {
      forecast_update(S, W, q.state.T, q.det + (size_t)q.det_start[d] * 7, q.det_n[d], row[1], start, q.match_iou_th,
                      false);
      __syncthreads();
      prev = d, start = false;
    }
    const size_t o = (size_t)row[3];
    const int n = forecast_extrap(S, (float)row[2], (float)row[4], (float)row[5], q.box_out + o * 4, q.score_out + o,
                                  q.label_out + o, q.track_out + o);
    if (threadIdx.x == 0) q.rows_out[f] = n;
  }
}

static inline bool state_ok(const SyForecastState& st) {
  return st.x && st.P && st.label && st.score && st.track && st.meta;
}

}  // namespace sy

using namespace sy;

extern "C" size_t sy_forecast_workspace_bytes(int32_t streams, int32_t max_tracks) {
  return streams > 0 && max_tracks > 0 ? (size_t)streams * max_tracks * kFcScratchWords * 4 : 0;
}

#define FC_STATE_CHECK(st, what)                                                                                   \
  SY_REQUIRE(state_ok(st), SY_EINVAL, what ": null state pointer");                                                \
  SY_REQUIRE((st).S > 0 && (st).S <= 65535, SY_EINVAL, what ": %d streams (1 to 65535)", (st).S);                  \
  SY_REQUIRE((st).T >= 1 && (st).T <= (1 << 20), SY_EINVAL, what ": max_tracks %d (1 to 2^20)", (st).T)

extern "C" int sy_forecast_update(const SyForecastUpdateDesc* d, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(d != nullptr, SY_EINVAL, "null descriptor");
  FC_STATE_CHECK(d->state, "forecast_update");
  SY_REQUIRE(d->det && d->count && d->dt && d->workspace, SY_EINVAL, "forecast_update: null pointer");
  SY_REQUIRE(d->max_det > 0, SY_EINVAL, "forecast_update: max_det %d", d->max_det);
  SY_REQUIRE(d->workspace_bytes >= sy_forecast_workspace_bytes(d->state.S, d->state.T), SY_EWORKSPACE,
             "forecast_update: workspace %zu < %zu", d->workspace_bytes, sy_forecast_workspace_bytes(d->state.S, d->state.T));
  forecast_update_kernel<<<d->state.S, kFcThreads, 0, stream>>>(*d);
  return launch_status("forecast_update_kernel");
}

extern "C" int sy_forecast_extrap(const SyForecastExtrapDesc* d, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(d != nullptr, SY_EINVAL, "null descriptor");
  FC_STATE_CHECK(d->state, "forecast_extrap");
  SY_REQUIRE(d->dt && d->img_wh && d->box_out && d->score_out && d->label_out && d->track_out && d->count_out, SY_EINVAL,
             "forecast_extrap: null pointer");
  forecast_extrap_kernel<<<d->state.S, kFcThreads, 0, stream>>>(*d);
  return launch_status("forecast_extrap_kernel");
}

extern "C" int sy_forecast_extrap_queries(const SyForecastExtrapQueriesDesc* d, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(d != nullptr, SY_EINVAL, "null descriptor");
  FC_STATE_CHECK(d->state, "forecast_extrap_queries");
  SY_REQUIRE(d->Q >= 1 && d->Q <= 65535, SY_EINVAL, "forecast_extrap_queries: %d queries per stream (1 to 65535)", d->Q);
  SY_REQUIRE(d->dt && d->n_query && d->img_wh && d->box_out && d->score_out && d->label_out && d->track_out &&
             d->count_out, SY_EINVAL, "forecast_extrap_queries: null pointer");
  forecast_extrap_queries_kernel<<<dim3(d->state.S, d->Q), kFcThreads, 0, stream>>>(*d);
  return launch_status("forecast_extrap_queries_kernel");
}

extern "C" int sy_forecast_sequences(const SyForecastSequencesDesc* d, sy_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SY_REQUIRE(d != nullptr, SY_EINVAL, "null descriptor");
  FC_STATE_CHECK(d->state, "forecast_sequences");
  SY_REQUIRE(d->det && d->det_start && d->det_n && d->frames && d->seq_frames && d->box_out && d->score_out &&
             d->label_out && d->track_out && d->rows_out && d->workspace, SY_EINVAL, "forecast_sequences: null pointer");
  SY_REQUIRE(d->workspace_bytes >= sy_forecast_workspace_bytes(d->state.S, d->state.T), SY_EWORKSPACE,
             "forecast_sequences: workspace %zu < %zu", d->workspace_bytes,
             sy_forecast_workspace_bytes(d->state.S, d->state.T));
  forecast_sequences_kernel<<<d->state.S, kFcThreads, 0, stream>>>(*d);
  return launch_status("forecast_sequences_kernel");
}
