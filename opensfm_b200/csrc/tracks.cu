// TRACKS: link pair matches into tracks on the device.
//
// Replaces tracking.create_tracks_manager (opensfm/tracking.py:72-150: a Python union-find keyed by
// (image, feature) tuples, one union per match, then _good_track, :238-244) and the two calls that bootstrap
// the reconstruction from its result, TracksManager::GetAllPairsConnectivity / GetAllCommonObservations
// (opensfm/src/map/src/tracks_manager.cc:285-350), for all image pairs at once.
//
// Nodes are features, node = image_offset[image] + feature; edges are the match rows.
//   build:  trk_link_edges   index check, touch, lock-free union-find (hook the larger root under the smaller
//                            with atomicCAS, path halving)
//           trk_labels       label = root = smallest node of the component: canonical, so the result does not
//                            depend on edge order or scheduling
//           radix sort of the touched nodes by label (stable: nodes ascending inside a label)
//           trk_node_info .. trk_emit   segments, the reference's filter, numbering by scan, output sorted by
//                            (track, image)
//   common: trk_pair_counts .. trk_pair_finish   every (track, image a < image b) keyed by the image pair, one
//                            radix sort, run lengths = connectivity
// The host reads back only counts (TrkCounts).
#include <thrust/iterator/counting_iterator.h>

#include <algorithm>
#include <cub/cub.cuh>
#include <vector>

#include "common.cuh"

namespace osfm {
namespace {

constexpr int TRK_THREADS = 256;
constexpr long long TRK_MAX_ITEMS = 2147483647LL;

struct TrkCounts {
  int err;                        // bit 0: image index outside [0, I), bit 1: feature index outside its image
  int num_tracks;
  int num_observations;
  unsigned long long first_bad;   // lowest match row with an error
};

// per sorted node: starts a segment / lies in an image with features / same image as its predecessor
struct TrkNode {
  int head, feat, dup;
};
struct TrkNodeSum {
  __host__ __device__ TrkNode operator()(const TrkNode& a, const TrkNode& b) const {
    return TrkNode{a.head + b.head, a.feat + b.feat, a.dup + b.dup};
  }
};
// per segment: is a track / its observations if it is
struct TrkSeg {
  int track, obs;
};
struct TrkSegSum {
  __host__ __device__ TrkSeg operator()(const TrkSeg& a, const TrkSeg& b) const {
    return TrkSeg{a.track + b.track, a.obs + b.obs};
  }
};

inline unsigned trk_blocks(long long n) { return (unsigned)((n + TRK_THREADS - 1) / TRK_THREADS); }

__global__ void trk_init(int n, int* __restrict__ parent, unsigned char* __restrict__ touched) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n) return;
  parent[v] = v;
  touched[v] = 0;
}

// Root of v.  parent[x] <= x always (hooks go from the larger root to the smaller one), and a non-root is only
// ever re-pointed to one of its ancestors, so concurrent halving keeps every chain valid and finite.
__device__ __forceinline__ int trk_find(int* parent, int v) {
  volatile int* vp = parent;
  int p = vp[v];
  while (p != v) {
    const int gp = vp[p];
    if (gp == p) return p;
    vp[v] = gp;
    v = gp;
    p = vp[v];
  }
  return v;
}

// last i in [0, n) with start[i] <= x (start ascending, start[0] <= x < start[n])
template <class T>
__device__ __forceinline__ int trk_owner(const T* __restrict__ start, int n, T x) {
  int lo = 0, hi = n;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (start[mid] <= x) lo = mid; else hi = mid;
  }
  return lo;
}

__global__ void trk_link_edges(long long E, const int2* __restrict__ matches, const long long* __restrict__ match_start,
                               int P, const int* __restrict__ pair_a, const int* __restrict__ pair_b, int I,
                               const int* __restrict__ img_off, int* parent, unsigned char* touched, TrkCounts* c) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const int p = trk_owner(match_start, P, e);
  const int a = pair_a[p], b = pair_b[p];
  const int2 m = matches[e];
  int err = 0;
  if (a < 0 || a >= I || b < 0 || b >= I) err = 1;
  else if (m.x < 0 || m.x >= img_off[a + 1] - img_off[a] || m.y < 0 || m.y >= img_off[b + 1] - img_off[b]) err = 2;
  if (err) {
    atomicOr(&c->err, err);
    atomicMin(&c->first_bad, (unsigned long long)e);
    return;
  }
  int u = img_off[a] + m.x, v = img_off[b] + m.y;
  touched[u] = 1;
  touched[v] = 1;
  while (true) {
    u = trk_find(parent, u);
    v = trk_find(parent, v);
    if (u == v) break;
    const int hi = max(u, v), lo = min(u, v);
    const int old = atomicCAS(&parent[hi], hi, lo);
    if (old == hi) break;
    u = old;   // hi was hooked meanwhile: carry on from its new parent
    v = lo;
  }
}

__global__ void trk_labels(int M, const int* __restrict__ nodes, int* parent, unsigned* __restrict__ label) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  label[i] = (unsigned)trk_find(parent, nodes[i]);
}

// i = 0..M (entry M is the zero that makes the exclusive scan end in the totals)
__global__ void trk_node_info(int M, const unsigned* __restrict__ label, const int* __restrict__ node, int I,
                              const int* __restrict__ img_off, const unsigned char* __restrict__ has_features,
                              int* __restrict__ img, TrkNode* __restrict__ info) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > M) return;
  if (i == M) { info[i] = TrkNode{0, 0, 0}; return; }
  const int im = trk_owner(img_off, I, node[i]);
  const bool head = i == 0 || label[i] != label[i - 1];
  const bool dup = !head && trk_owner(img_off, I, node[i - 1]) == im;
  img[i] = im;
  info[i] = TrkNode{head ? 1 : 0, has_features[im] ? 1 : 0, dup ? 1 : 0};
}

__global__ void trk_segments(int M, const TrkNode* __restrict__ scan, int* __restrict__ seg_first) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  if (scan[i + 1].head != scan[i].head) seg_first[scan[i].head] = i;
  if (i == 0) seg_first[scan[M].head] = M;
}

// _good_track (tracking.py:238-244) over EVERY node of the component, and at least one node to output
__global__ void trk_filter(int M, const TrkNode* __restrict__ scan, const int* __restrict__ seg_first, int min_length,
                           TrkSeg* __restrict__ seg) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s > M) return;
  TrkSeg r{0, 0};
  if (s < scan[M].head) {
    const int b = seg_first[s], e = seg_first[s + 1];
    const int kept = scan[e].feat - scan[b].feat;
    if (e - b >= min_length && scan[e].dup == scan[b].dup && kept > 0) r = TrkSeg{1, kept};
  }
  seg[s] = r;
}

__global__ void trk_emit(int M, const TrkNode* __restrict__ scan, const TrkSeg* __restrict__ seg_scan,
                         const int* __restrict__ seg_first, const int* __restrict__ node, const int* __restrict__ img,
                         const int* __restrict__ img_off, int* __restrict__ obs_track, int* __restrict__ obs_image,
                         int* __restrict__ obs_feature, long long* __restrict__ track_start, TrkCounts* c) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  if (i == 0) {
    c->num_tracks = seg_scan[M].track;
    c->num_observations = seg_scan[M].obs;
    track_start[seg_scan[M].track] = seg_scan[M].obs;
  }
  const int s = scan[i + 1].head - 1;
  if (seg_scan[s + 1].track == seg_scan[s].track) return;
  const int b = seg_first[s];
  if (i == b) track_start[seg_scan[s].track] = seg_scan[s].obs;
  if (scan[i + 1].feat == scan[i].feat) return;
  const int pos = seg_scan[s].obs + (scan[i].feat - scan[b].feat);
  obs_track[pos] = seg_scan[s].track;
  obs_image[pos] = img[i];
  obs_feature[pos] = node[i] - img_off[img[i]];
}

// a track of L observations has one observation per image, so it joins L (L - 1) / 2 image pairs
__global__ void trk_pair_counts(int T, const long long* __restrict__ track_start, long long* __restrict__ cnt) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t > T) return;
  long long n = 0;
  if (t < T) {
    const long long L = track_start[t + 1] - track_start[t];
    n = L * (L - 1) / 2;
  }
  cnt[t] = n;
}

// r -> (track, a < b): key = image_a * I + image_b, payload = the two observation indices
__global__ void trk_emit_pairs(long long R, int T, const long long* __restrict__ pair_off,
                               const long long* __restrict__ track_start, const int* __restrict__ obs_image, int I,
                               unsigned long long* __restrict__ key, unsigned long long* __restrict__ val) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  const int t = trk_owner(pair_off, T, r);
  const long long k = r - pair_off[t];
  const long long o = track_start[t], L = track_start[t + 1] - o;
  // rows (0,1) .. (0,L-1), (1,2) ..: row i starts at i (2L - i - 1) / 2
  const double w = (double)(2 * L - 1);
  long long i = (long long)((w - sqrt(w * w - 8.0 * (double)k)) * 0.5);
  i = max(0LL, min(i, L - 2));
  while (i > 0 && i * (2 * L - i - 1) / 2 > k) --i;
  while ((i + 1) * (2 * L - i - 2) / 2 <= k) ++i;
  const long long j = i + 1 + (k - i * (2 * L - i - 1) / 2);
  const unsigned long long oa = (unsigned long long)(o + i), ob = (unsigned long long)(o + j);
  key[r] = (unsigned long long)obs_image[oa] * (unsigned long long)I + (unsigned long long)obs_image[ob];
  val[r] = (oa << 32) | ob;
}

__global__ void trk_pair_heads(long long R, const unsigned long long* __restrict__ key, unsigned char* __restrict__ head) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  head[r] = (r == 0 || key[r] != key[r - 1]) ? 1 : 0;
}

// n = max(Q + 1, R) threads
__global__ void trk_pair_finish(long long R, int Q, int I, const unsigned long long* __restrict__ key,
                                const unsigned long long* __restrict__ val, long long* __restrict__ pair_start,
                                int* __restrict__ pair_a, int* __restrict__ pair_b, long long* __restrict__ common_a,
                                long long* __restrict__ common_b) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r < Q) {
    const unsigned long long k = key[pair_start[r]];
    pair_a[r] = (int)(k / (unsigned long long)I);
    pair_b[r] = (int)(k % (unsigned long long)I);
  } else if (r == Q) {
    pair_start[Q] = R;
  }
  if (r < R) {
    common_a[r] = (long long)(val[r] >> 32);
    common_b[r] = (long long)(val[r] & 0xffffffffULL);
  }
}

int trk_bits(unsigned long long max_value) {
  int b = 1;
  while (b < 64 && (max_value >> b)) ++b;
  return b;
}

struct Tracks : DeviceStream<4> {   // events: build start / end, common start / end
  bool built = false, common_built = false, timed_build = false, timed_common = false;
  int I = 0, T = 0, Q = 0;
  long long nobs = 0, R = 0;

  DevBuf<int> d_img_off, d_pair_a, d_pair_b, d_parent, d_nodes, d_nodes_sorted, d_img, d_seg_first;
  DevBuf<long long> d_match_start;
  DevBuf<int2> d_matches;
  DevBuf<unsigned char> d_has_features, d_touched, d_tmp;
  DevBuf<unsigned> d_label, d_label_sorted;
  DevBuf<TrkNode> d_info, d_scan;
  DevBuf<TrkSeg> d_seg, d_seg_scan;
  DevBuf<int> d_obs_track, d_obs_image, d_obs_feature;
  DevBuf<long long> d_track_start;
  DevBuf<TrkCounts> d_counts;
  DevBuf<int> d_num_selected;
  // common tracks
  DevBuf<long long> d_pair_cnt, d_pair_off, d_pair_start;
  DevBuf<unsigned long long> d_key, d_val, d_key_sorted, d_val_sorted;
  DevBuf<unsigned char> d_head;
  DevBuf<int> d_cpair_a, d_cpair_b;
  PinnedBuf<TrkCounts> h_counts;
  PinnedBuf<long long> h_ll;

  explicit Tracks(int dev) : DeviceStream(dev) {
    d_counts.reserve(1);
    d_num_selected.reserve(1);
    h_counts.reserve(1);
    h_ll.reserve(1);
  }

  const TrkCounts& read_counts() {
    OSFM_CUDA(cudaMemcpyAsync(h_counts.p, d_counts.p, sizeof(TrkCounts), cudaMemcpyDeviceToHost, stream));
    OSFM_CUDA(cudaStreamSynchronize(stream));
    return *h_counts.p;
  }

  void build(int num_images, const int32_t* num_features, const uint8_t* has_features, int64_t num_pairs,
             const int32_t* pair_a, const int32_t* pair_b, const int64_t* match_start, const int32_t* matches,
             int min_length, int64_t* num_tracks, int64_t* num_observations);
  void common(int64_t* num_pairs, int64_t* num_common);
};

void Tracks::build(int num_images, const int32_t* num_features, const uint8_t* has_features, int64_t num_pairs,
                   const int32_t* pair_a, const int32_t* pair_b, const int64_t* match_start, const int32_t* matches,
                   int min_length, int64_t* num_tracks, int64_t* num_observations) {
  built = common_built = timed_build = timed_common = false;
  if (num_images < 0 || num_pairs < 0 || num_pairs > TRK_MAX_ITEMS) throw ArgError("bad tracks sizes");
  if (!num_tracks || !num_observations) throw ArgError("null outputs");
  if ((num_images > 0 && (!num_features || !has_features)) || (num_pairs > 0 && (!pair_a || !pair_b)) || !match_start)
    throw ArgError("null arrays");
  std::vector<int> off((size_t)num_images + 1);
  long long N = 0;
  for (int i = 0; i < num_images; ++i) {
    if (num_features[i] < 0) throw ArgError("negative feature count of image " + std::to_string(i));
    off[i] = (int)N;
    N += num_features[i];
    if (N > TRK_MAX_ITEMS)
      throw ArgError("tracks: more than 2^31 - 1 features in all (reached at image " + std::to_string(i) + ")");
  }
  off[num_images] = (int)N;
  if (match_start[0] != 0) throw ArgError("match_start[0] must be 0");
  for (int64_t p = 0; p < num_pairs; ++p)
    if (match_start[p + 1] < match_start[p]) throw ArgError("match_start must not decrease (pair " + std::to_string(p) + ")");
  const long long E = match_start[num_pairs];
  if (E > TRK_MAX_ITEMS) throw ArgError("tracks: more than 2^31 - 1 match rows (" + std::to_string(E) + ")");
  if (E > 0 && !matches) throw ArgError("null matches");
  I = num_images;
  T = 0;
  nobs = 0;

  upload(d_img_off, off.data(), off.size());
  upload(d_has_features, has_features, (size_t)num_images);
  upload(d_pair_a, pair_a, (size_t)num_pairs);
  upload(d_pair_b, pair_b, (size_t)num_pairs);
  upload(d_match_start, reinterpret_cast<const long long*>(match_start), (size_t)num_pairs + 1);
  upload(d_matches, reinterpret_cast<const int2*>(matches), (size_t)E);
  OSFM_CUDA(cudaEventRecord(ev[0], stream));   // the device time is that of the kernels, not of the uploads
  TrkCounts zero{0, 0, 0, ~0ULL};
  *h_counts.p = zero;
  OSFM_CUDA(cudaMemcpyAsync(d_counts.p, h_counts.p, sizeof(TrkCounts), cudaMemcpyHostToDevice, stream));
  d_track_start.reserve(1);
  OSFM_CUDA(cudaMemsetAsync(d_track_start.p, 0, sizeof(long long), stream));

  int M = 0;
  if (E > 0 && N > 0) {
    d_parent.reserve((size_t)N);
    d_touched.reserve((size_t)N);
    d_nodes.reserve((size_t)N);
    trk_init<<<trk_blocks(N), TRK_THREADS, 0, stream>>>((int)N, d_parent.p, d_touched.p);
    OSFM_LAUNCH_CHECK();
    trk_link_edges<<<trk_blocks(E), TRK_THREADS, 0, stream>>>(E, d_matches.p, d_match_start.p, (int)num_pairs,
                                                              d_pair_a.p, d_pair_b.p, I, d_img_off.p, d_parent.p,
                                                              d_touched.p, d_counts.p);
    OSFM_LAUNCH_CHECK();
    thrust::counting_iterator<int> ids(0);
    size_t bytes = 0;
    OSFM_CUDA(cub::DeviceSelect::Flagged(nullptr, bytes, ids, d_touched.p, d_nodes.p, d_num_selected.p, (int)N, stream));
    d_tmp.reserve(bytes);
    OSFM_CUDA(cub::DeviceSelect::Flagged(d_tmp.p, bytes, ids, d_touched.p, d_nodes.p, d_num_selected.p, (int)N, stream));
    OSFM_CUDA(cudaMemcpyAsync(h_ll.p, d_num_selected.p, sizeof(int), cudaMemcpyDeviceToHost, stream));
  } else if (E > 0) {
    // no image has a feature: every row is out of range
    trk_link_edges<<<trk_blocks(E), TRK_THREADS, 0, stream>>>(E, d_matches.p, d_match_start.p, (int)num_pairs,
                                                              d_pair_a.p, d_pair_b.p, I, d_img_off.p, nullptr, nullptr,
                                                              d_counts.p);
    OSFM_LAUNCH_CHECK();
  }
  const TrkCounts c = read_counts();
  if (c.err) {
    const long long e = (long long)c.first_bad;
    const int64_t p = std::upper_bound(match_start, match_start + num_pairs + 1, (int64_t)e) - match_start - 1;
    char buf[384];
    if (c.err & 1 && (pair_a[p] < 0 || pair_a[p] >= I || pair_b[p] < 0 || pair_b[p] >= I)) {
      snprintf(buf, sizeof(buf), "tracks: pair %lld names images (%d, %d), outside [0, %d)", (long long)p, pair_a[p],
               pair_b[p], I);
    } else {
      const int fa = matches[2 * e], fb = matches[2 * e + 1];
      const bool first = fa < 0 || fa >= num_features[pair_a[p]];
      snprintf(buf, sizeof(buf),
               "tracks: match row %lld (row %lld of pair %lld, images %d and %d): feature index %d is outside [0, %d) "
               "of image %d",
               e, e - (long long)match_start[p], (long long)p, pair_a[p], pair_b[p], first ? fa : fb,
               num_features[first ? pair_a[p] : pair_b[p]], first ? pair_a[p] : pair_b[p]);
    }
    throw std::runtime_error(buf);
  }
  if (E > 0 && N > 0) M = *reinterpret_cast<int*>(h_ll.p);

  if (M > 0) {
    d_label.reserve((size_t)M);
    d_label_sorted.reserve((size_t)M);
    d_nodes_sorted.reserve((size_t)M);
    d_img.reserve((size_t)M);
    d_seg_first.reserve((size_t)M + 1);
    d_info.reserve((size_t)M + 1);
    d_scan.reserve((size_t)M + 1);
    d_seg.reserve((size_t)M + 1);
    d_seg_scan.reserve((size_t)M + 1);
    d_obs_track.reserve((size_t)M);
    d_obs_image.reserve((size_t)M);
    d_obs_feature.reserve((size_t)M);
    d_track_start.reserve((size_t)M + 1);
    trk_labels<<<trk_blocks(M), TRK_THREADS, 0, stream>>>(M, d_nodes.p, d_parent.p, d_label.p);
    OSFM_LAUNCH_CHECK();
    const int bits = trk_bits((unsigned long long)N - 1);
    size_t bytes = 0, b2 = 0, b3 = 0;
    OSFM_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, bytes, d_label.p, d_label_sorted.p, d_nodes.p, d_nodes_sorted.p,
                                              M, 0, bits, stream));
    OSFM_CUDA(cub::DeviceScan::ExclusiveScan(nullptr, b2, d_info.p, d_scan.p, TrkNodeSum(), TrkNode{0, 0, 0}, M + 1,
                                             stream));
    OSFM_CUDA(cub::DeviceScan::ExclusiveScan(nullptr, b3, d_seg.p, d_seg_scan.p, TrkSegSum(), TrkSeg{0, 0}, M + 1,
                                             stream));
    bytes = std::max(bytes, std::max(b2, b3));
    d_tmp.reserve(bytes);
    OSFM_CUDA(cub::DeviceRadixSort::SortPairs(d_tmp.p, bytes, d_label.p, d_label_sorted.p, d_nodes.p, d_nodes_sorted.p,
                                              M, 0, bits, stream));
    trk_node_info<<<trk_blocks(M + 1), TRK_THREADS, 0, stream>>>(M, d_label_sorted.p, d_nodes_sorted.p, I, d_img_off.p,
                                                                 d_has_features.p, d_img.p, d_info.p);
    OSFM_LAUNCH_CHECK();
    OSFM_CUDA(cub::DeviceScan::ExclusiveScan(d_tmp.p, bytes, d_info.p, d_scan.p, TrkNodeSum(), TrkNode{0, 0, 0}, M + 1,
                                             stream));
    trk_segments<<<trk_blocks(M), TRK_THREADS, 0, stream>>>(M, d_scan.p, d_seg_first.p);
    OSFM_LAUNCH_CHECK();
    trk_filter<<<trk_blocks(M + 1), TRK_THREADS, 0, stream>>>(M, d_scan.p, d_seg_first.p, min_length, d_seg.p);
    OSFM_LAUNCH_CHECK();
    OSFM_CUDA(cub::DeviceScan::ExclusiveScan(d_tmp.p, bytes, d_seg.p, d_seg_scan.p, TrkSegSum(), TrkSeg{0, 0}, M + 1,
                                             stream));
    trk_emit<<<trk_blocks(M), TRK_THREADS, 0, stream>>>(M, d_scan.p, d_seg_scan.p, d_seg_first.p, d_nodes_sorted.p,
                                                        d_img.p, d_img_off.p, d_obs_track.p, d_obs_image.p,
                                                        d_obs_feature.p, d_track_start.p, d_counts.p);
    OSFM_LAUNCH_CHECK();
    OSFM_CUDA(cudaEventRecord(ev[1], stream));
    const TrkCounts r = read_counts();
    T = r.num_tracks;
    nobs = r.num_observations;
  } else {
    OSFM_CUDA(cudaEventRecord(ev[1], stream));
    OSFM_CUDA(cudaStreamSynchronize(stream));
  }
  *num_tracks = T;
  *num_observations = nobs;
  built = timed_build = true;
}

void Tracks::common(int64_t* num_pairs, int64_t* num_common) {
  if (!built) throw std::runtime_error("tracks: osfm_tracks_common needs a successful osfm_tracks_build");
  if (!num_pairs || !num_common) throw ArgError("null outputs");
  common_built = timed_common = false;
  Q = 0;
  R = 0;
  OSFM_CUDA(cudaEventRecord(ev[2], stream));
  if (T > 0) {
    d_pair_cnt.reserve((size_t)T + 1);
    d_pair_off.reserve((size_t)T + 1);
    trk_pair_counts<<<trk_blocks(T + 1), TRK_THREADS, 0, stream>>>(T, d_track_start.p, d_pair_cnt.p);
    OSFM_LAUNCH_CHECK();
    size_t bytes = 0;
    OSFM_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, bytes, d_pair_cnt.p, d_pair_off.p, T + 1, stream));
    d_tmp.reserve(bytes);
    OSFM_CUDA(cub::DeviceScan::ExclusiveSum(d_tmp.p, bytes, d_pair_cnt.p, d_pair_off.p, T + 1, stream));
    OSFM_CUDA(cudaMemcpyAsync(h_ll.p, d_pair_off.p + T, sizeof(long long), cudaMemcpyDeviceToHost, stream));
    OSFM_CUDA(cudaStreamSynchronize(stream));
    R = *h_ll.p;
  }
  if (R > TRK_MAX_ITEMS)
    throw std::runtime_error("tracks: " + std::to_string(R) + " common observations, more than 2^31 - 1");
  if (R > 0) {
    const long long qmax = std::min<long long>(R, (long long)I * (I - 1) / 2);
    const int n = (int)R;
    const int bits = trk_bits((unsigned long long)I * (unsigned long long)I - 1);
    thrust::counting_iterator<long long> rows(0);
    size_t bytes = 0, b2 = 0;
    try {
      d_key.reserve((size_t)R);
      d_val.reserve((size_t)R);
      d_key_sorted.reserve((size_t)R);
      d_val_sorted.reserve((size_t)R);
      d_head.reserve((size_t)R);
      d_pair_start.reserve((size_t)qmax + 1);
      d_cpair_a.reserve((size_t)qmax);
      d_cpair_b.reserve((size_t)qmax);
      OSFM_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, bytes, d_key.p, d_key_sorted.p, d_val.p, d_val_sorted.p, n, 0,
                                                bits, stream));
      OSFM_CUDA(cub::DeviceSelect::Flagged(nullptr, b2, rows, d_head.p, d_pair_start.p, d_num_selected.p, n, stream));
      bytes = std::max(bytes, b2);
      d_tmp.reserve(bytes);
    } catch (const CudaError& e) {
      cudaGetLastError();   // a failed cudaMalloc is not sticky; keep it from failing the next launch check
      throw CudaError("tracks: no device memory for the " + std::to_string(R) +
                      " common observations of all image pairs (about " + std::to_string((33 * R) >> 20) +
                      " MB): " + e.what());
    }
    trk_emit_pairs<<<trk_blocks(R), TRK_THREADS, 0, stream>>>(R, T, d_pair_off.p, d_track_start.p, d_obs_image.p, I,
                                                              d_key.p, d_val.p);
    OSFM_LAUNCH_CHECK();
    OSFM_CUDA(cub::DeviceRadixSort::SortPairs(d_tmp.p, bytes, d_key.p, d_key_sorted.p, d_val.p, d_val_sorted.p, n, 0,
                                              bits, stream));
    trk_pair_heads<<<trk_blocks(R), TRK_THREADS, 0, stream>>>(R, d_key_sorted.p, d_head.p);
    OSFM_LAUNCH_CHECK();
    OSFM_CUDA(cub::DeviceSelect::Flagged(d_tmp.p, bytes, rows, d_head.p, d_pair_start.p, d_num_selected.p, n, stream));
    OSFM_CUDA(cudaMemcpyAsync(h_ll.p, d_num_selected.p, sizeof(int), cudaMemcpyDeviceToHost, stream));
    OSFM_CUDA(cudaStreamSynchronize(stream));
    Q = *reinterpret_cast<int*>(h_ll.p);
    // the sort's input buffers are free again: they take the observation indices as int64
    trk_pair_finish<<<trk_blocks(std::max<long long>(R, Q + 1)), TRK_THREADS, 0, stream>>>(
        R, Q, I, d_key_sorted.p, d_val_sorted.p, d_pair_start.p, d_cpair_a.p, d_cpair_b.p,
        reinterpret_cast<long long*>(d_key.p), reinterpret_cast<long long*>(d_val.p));
    OSFM_LAUNCH_CHECK();
  }
  OSFM_CUDA(cudaEventRecord(ev[3], stream));
  OSFM_CUDA(cudaStreamSynchronize(stream));
  *num_pairs = Q;
  *num_common = R;
  common_built = timed_common = true;
}

}  // namespace
}  // namespace osfm

struct osfm_tracks : osfm::Handle<osfm::Tracks> {
  using Handle::Handle;
  static constexpr const char* null_message = "null tracks";
};

extern "C" {

int osfm_tracks_create(int device, osfm_tracks** out) { return osfm::create_handle(device, out); }
int osfm_tracks_destroy(osfm_tracks* t) { return osfm::destroy_handle(t); }

int osfm_tracks_build(osfm_tracks* t, int num_images, const int32_t* num_features, const uint8_t* has_features,
                      int64_t num_pairs, const int32_t* pair_a, const int32_t* pair_b, const int64_t* match_start,
                      const int32_t* matches, int min_length, int64_t* num_tracks, int64_t* num_observations) {
  return osfm::with_handle(t, [&](osfm::Tracks& K) {
    K.build(num_images, num_features, has_features, num_pairs, pair_a, pair_b, match_start, matches, min_length,
            num_tracks, num_observations);
  });
}

int osfm_tracks_get(osfm_tracks* t, int32_t* obs_track, int32_t* obs_image, int32_t* obs_feature,
                    int64_t* track_start) {
  return osfm::with_handle(t, [&](osfm::Tracks& K) {
    if (!K.built) throw std::runtime_error("tracks: osfm_tracks_get needs a successful osfm_tracks_build");
    if (!track_start || (K.nobs > 0 && (!obs_track || !obs_image || !obs_feature))) throw osfm::ArgError("null outputs");
    K.download(obs_track, K.d_obs_track.p, (size_t)K.nobs);
    K.download(obs_image, K.d_obs_image.p, (size_t)K.nobs);
    K.download(obs_feature, K.d_obs_feature.p, (size_t)K.nobs);
    K.download(reinterpret_cast<long long*>(track_start), K.d_track_start.p, (size_t)K.T + 1);
    OSFM_CUDA(cudaStreamSynchronize(K.stream));
  });
}

int osfm_tracks_common(osfm_tracks* t, int64_t* num_pairs, int64_t* num_common) {
  return osfm::with_handle(t, [&](osfm::Tracks& K) { K.common(num_pairs, num_common); });
}

int osfm_tracks_get_common(osfm_tracks* t, int32_t* pair_a, int32_t* pair_b, int64_t* pair_start,
                           int64_t* common_obs_a, int64_t* common_obs_b) {
  return osfm::with_handle(t, [&](osfm::Tracks& K) {
    if (!K.common_built)
      throw std::runtime_error("tracks: osfm_tracks_get_common needs a successful osfm_tracks_common");
    if (!pair_start || (K.Q > 0 && (!pair_a || !pair_b)) || (K.R > 0 && (!common_obs_a || !common_obs_b)))
      throw osfm::ArgError("null outputs");
    if (K.R == 0) {
      pair_start[0] = 0;
      return;
    }
    K.download(pair_a, K.d_cpair_a.p, (size_t)K.Q);
    K.download(pair_b, K.d_cpair_b.p, (size_t)K.Q);
    K.download(reinterpret_cast<long long*>(pair_start), K.d_pair_start.p, (size_t)K.Q + 1);
    K.download(reinterpret_cast<long long*>(common_obs_a), reinterpret_cast<long long*>(K.d_key.p), (size_t)K.R);
    K.download(reinterpret_cast<long long*>(common_obs_b), reinterpret_cast<long long*>(K.d_val.p), (size_t)K.R);
    OSFM_CUDA(cudaStreamSynchronize(K.stream));
  });
}

int osfm_tracks_last_device_ms(osfm_tracks* t, float* ms_build, float* ms_common) {
  return osfm::with_handle(t, [&](osfm::Tracks& K) {
    if (ms_build) {
      *ms_build = 0.f;
      if (K.timed_build) OSFM_CUDA(cudaEventElapsedTime(ms_build, K.ev[0], K.ev[1]));
    }
    if (ms_common) {
      *ms_common = 0.f;
      if (K.timed_common) OSFM_CUDA(cudaEventElapsedTime(ms_common, K.ev[2], K.ev[3]));
    }
  });
}

}  // extern "C"
