// ORACLE (test infrastructure, not product code): C entry points of oracle/_ref/libref.so.
//
// libref.so = the reference's OWN translation units, compiled UNMODIFIED from where they lie under /root/reference
// (src/ORBExtractor.cpp, CamModelGeneral.cpp, Frame.cpp, ORBMatcher.cpp, KeyFrame.cpp, MapPoint.cpp, Map.cpp, KeyFrameDatabase.cpp and
// ThirdParty/DBoW2/DBoW2/*.cpp) against the cv:: shim in oracle/cvshim (no OpenCV C++ exists in this container), plus this file.
// This file holds only (1) flat C wrappers that call the reference classes the way the reference's own callers do (file:line cited), on
// objects built from flat arrays by oracle/ref_scene.cpp (which libdropin.so shares, so both harnesses check the same scenes),
// (2) the few caller-side lines of src/System.cpp that cannot be compiled here (System.cpp needs Pangolin): the map loop of
// CreateUndistortRectifyMap (:301-324) and the five cv::remap calls (:327-355), and (3) two optional PINS of behaviour the reference leaves to
// its environment:
//   PIN_ALLOC   std::list<ExtractorNode> nodes come from a monotonic arena, so the reference's `sort(pair<int,ExtractorNode*>)`
//               tie-break by heap address (src/ORBExtractor.cpp:658) is "later-created node first" -- the order the oracle defines;
//   PIN_SINCOS  sincosf (what gcc emits for cos/sin at src/ORBExtractor.cpp:83-84) is the fp64 det_sincos of oracle/cvprim.h instead
//               of glibc's, which is not correctly rounded.
// With both pins the reference code is deterministic and the tests require oracle == libref bit for bit; without them the tests
// QUANTIFY how far a stock glibc build drifts (tests/test_oracle_ref.py).
#include <dlfcn.h>
#include <sys/mman.h>
#include <atomic>
#include <cstring>
#include <mutex>
#include <new>
#include <thread>
#include <vector>

#include "Converter.h"
#include "ORBExtractor.h"
#include "ORBMatcher.h"
#include "ref_scene.h"

using namespace scene;

// ------------------------------------------------------------------------------------------------- pins
enum { PIN_ALLOC = 1, PIN_SINCOS = 2 };
static std::atomic<int> g_pins(0);

static const size_t kNodeBytes = sizeof(std::_List_node<ExtractorNode>);
static const size_t kArenaBytes = (size_t)4 << 30;   // virtual reservation only (MAP_NORESERVE)
static char* g_arena = nullptr;
static std::atomic<size_t> g_arenaUsed(0);
static std::once_flag g_arenaOnce;
static void arena_init() {
    void* p = mmap(nullptr, kArenaBytes, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
    g_arena = (p == MAP_FAILED) ? nullptr : (char*)p;
}
static inline bool in_arena(const void* p) { return g_arena && (const char*)p >= g_arena && (const char*)p < g_arena + kArenaBytes; }
static inline void* ref_alloc(size_t n) {
    if ((g_pins.load(std::memory_order_relaxed) & PIN_ALLOC) && n == kNodeBytes) {
        std::call_once(g_arenaOnce, arena_init);
        if (g_arena) {
            const size_t off = g_arenaUsed.fetch_add((n + 15) & ~(size_t)15);
            if (off + n <= kArenaBytes) return g_arena + off;
        }
    }
    void* p = std::malloc(n ? n : 1);
    if (!p) throw std::bad_alloc();
    return p;
}
static inline void ref_free(void* p) { if (p && !in_arena(p)) std::free(p); }
// replaced inside this shared object only (linked with -Bsymbolic; the library is loaded RTLD_LOCAL)
void* operator new(size_t n) { return ref_alloc(n); }
void* operator new[](size_t n) { return ref_alloc(n); }
void operator delete(void* p) noexcept { ref_free(p); }
void operator delete[](void* p) noexcept { ref_free(p); }
void operator delete(void* p, size_t) noexcept { ref_free(p); }
void operator delete[](void* p, size_t) noexcept { ref_free(p); }

extern "C" void sincosf(float x, float* s, float* c) {
    if (g_pins.load(std::memory_order_relaxed) & PIN_SINCOS) { orc::det_sincosf(x, s, c); return; }
    typedef void (*fn_t)(float, float*, float*);
    static fn_t real = (fn_t)dlsym(RTLD_NEXT, "sincosf");
    real(x, s, c);
}

extern "C" {

void ref_set_pins(int mask) { g_pins.store(mask); }
int ref_get_pins() { return g_pins.load(); }
size_t ref_arena_used() { return g_arenaUsed.load(); }

void ref_set_camera(const RefCam* cp) { set_camera(cp); }
float ref_cos_fov_th() { return CamModelGeneral::GetCamera()->GetCosFovTh(); }

// System::CreateUndistortRectifyMap, src/System.cpp:301-324 (the loop around CamModelGeneral::CubemapToFisheye)
void ref_build_maps(float* map1, float* map2) {
    CamModelGeneral* cam = CamModelGeneral::GetCamera();
    const int width3 = cam->GetCubeFaceWidth() * 3, height3 = cam->GetCubeFaceHeight() * 3;
    cv::Mat mMap1(height3, width3, CV_32F, map1), mMap2(height3, width3, CV_32F, map2);
    mMap1.setTo(0); mMap2.setTo(0);
    const int Iw = cam->GetFisheyeWidth(), Ih = cam->GetFisheyeHeight();
    for (int y = 0; y < height3; ++y)
        for (int x = 0; x < width3; ++x) {
            double u, v;
            cam->CubemapToFisheye(u, v, static_cast<double>(x), static_cast<double>(y));
            if (u < 0 || v < 0 || u >= Iw || v >= Ih) continue;
            mMap1.at<float>(y, x) = static_cast<float>(u);
            mMap2.at<float>(y, x) = static_cast<float>(v);
        }
}
void ref_cubemap_to_fisheye(double up, double vp, double* uf, double* vf) { CamModelGeneral::GetCamera()->CubemapToFisheye(*uf, *vf, up, vp); }

// System::CvtFisheyeToCubeMap_reverseQuery_withInterpolation, src/System.cpp:327-355: five cv::remap calls on face ROIs
static void warp_into(cv::Mat& cubemapImg, const cv::Mat& fisheyeImg, const cv::Mat& mMap1, const cv::Mat& mMap2) {
    const int width = CamModelGeneral::GetCamera()->GetCubeFaceWidth(), height = CamModelGeneral::GetCamera()->GetCubeFaceHeight();
    const int r0[5] = {height, height, height, 0, 2 * height}, c0[5] = {width, 0, 2 * width, width, width};   // front, left, right, upper, lower
    for (int f = 0; f < 5; f++) {
        cv::Mat dst = cubemapImg.rowRange(r0[f], r0[f] + height).colRange(c0[f], c0[f] + width);
        cv::remap(fisheyeImg, dst, mMap1.rowRange(r0[f], r0[f] + height).colRange(c0[f], c0[f] + width),
                  mMap2.rowRange(r0[f], r0[f] + height).colRange(c0[f], c0[f] + width), cv::INTER_LINEAR, cv::BORDER_CONSTANT, cv::Scalar());
    }
}
void ref_warp(const uint8_t* fisheye, const float* map1, const float* map2, uint8_t* canvas) {
    CamModelGeneral* cam = CamModelGeneral::GetCamera();
    const int W3 = cam->GetCubeFaceWidth() * 3, H3 = cam->GetCubeFaceHeight() * 3;
    cv::Mat cub(H3, W3, CV_8UC1, canvas), fe(cam->GetFisheyeHeight(), cam->GetFisheyeWidth(), CV_8UC1, (void*)fisheye);
    cv::Mat m1(H3, W3, CV_32F, (void*)map1), m2(H3, W3, CV_32F, (void*)map2);
    warp_into(cub, fe, m1, m2);
}

// ---- ORBextractor (include/ORBExtractor.h:49-116), called like Frame::ExtractORB does (src/Frame.cpp:178-181)
struct RefOrb { ORBextractor* ex; std::vector<cv::KeyPoint> kps; cv::Mat desc; };
void* ref_orb_create(int nfeatures, float scaleFactor, int nlevels, int iniTh, int minTh) {
    RefOrb* h = new RefOrb; h->ex = new ORBextractor(nfeatures, scaleFactor, nlevels, iniTh, minTh); return h;
}
void ref_orb_destroy(void* hv) { RefOrb* h = (RefOrb*)hv; delete h->ex; delete h; }
int ref_orb_extract(void* hv, const uint8_t* img, int cols, int rows, const uint8_t* mask) {
    RefOrb* h = (RefOrb*)hv;
    cv::Mat im(rows, cols, CV_8UC1, (void*)img), mk(rows, cols, CV_8UC1, (void*)mask);
    (*h->ex)(im, mk, h->kps, h->desc);
    return (int)h->kps.size();
}
void ref_orb_result(void* hv, cv::KeyPoint* kps, uint8_t* desc) {
    RefOrb* h = (RefOrb*)hv;
    static_assert(sizeof(cv::KeyPoint) == 28, "cv::KeyPoint layout");
    const size_t n = h->kps.size();
    if (!n) return;
    std::memcpy((void*)kps, h->kps.data(), n * sizeof(cv::KeyPoint));
    for (size_t i = 0; i < n; i++) std::memcpy(desc + 32 * i, h->desc.ptr<uchar>((int)i), 32);
}
void ref_orb_level_size(void* hv, int level, int* w, int* hh) { const cv::Mat& L = ((RefOrb*)hv)->ex->mvImagePyramid[level]; *w = L.cols; *hh = L.rows; }
void ref_orb_level_image(void* hv, int level, uint8_t* out) {
    const cv::Mat& L = ((RefOrb*)hv)->ex->mvImagePyramid[level];
    for (int y = 0; y < L.rows; y++) std::memcpy(out + (size_t)y * L.cols, L.ptr<uchar>(y), (size_t)L.cols);
}

// ---- Frame (src/Frame.cpp:104-156): extraction + ComputeKeyPointRays (:746-760) + AssignFeaturesToGrid (:158-176), exactly as Tracking builds it
struct RefFrame { Frame* F; };
void* ref_frame_from_image(void* orb, const uint8_t* img, const uint8_t* mask, int rows, int cols) {
    RefOrb* h = (RefOrb*)orb;
    cv::Mat im(rows, cols, CV_8UC1, (void*)img), mk(rows, cols, CV_8UC1, (void*)mask);
    Frame::mbInitialComputations = true;   // grid geometry follows this image size (src/Frame.cpp:141-152)
    RefFrame* f = new RefFrame; f->F = new Frame(im, mk, 0.0, h->ex, static_cast<ORBVocabulary*>(NULL));
    return f;
}
void ref_frame_destroy(void* fv) { RefFrame* f = (RefFrame*)fv; delete f->F; delete f; }
int ref_frame_n(void* fv) { return ((RefFrame*)fv)->F->N; }
void ref_frame_get(void* fv, KpPOD* kps, uint8_t* desc, float* rays, int32_t* gridCount) {
    const Frame& F = *((RefFrame*)fv)->F;
    read_frame(F, F.N, kps, desc, rays, gridCount);
}
// grid cell contents in the reference's order: mGrid[face][col][row] (include/Frame.h:129)
int ref_frame_grid_cell(void* fv, int face, int col, int row, int32_t* idx, int cap) {
    const std::vector<size_t>& v = ((RefFrame*)fv)->F->mGrid[face][col][row];
    for (size_t i = 0; i < v.size() && (int)i < cap; i++) idx[i] = (int32_t)v[i];
    return (int)v.size();
}
// Frame::GetFeaturesInArea (src/Frame.cpp:251-716)
int ref_frame_features_in_area(void* fv, float x, float y, float r, int minLevel, int maxLevel, int32_t* idx, int cap) {
    const std::vector<size_t> v = ((RefFrame*)fv)->F->GetFeaturesInArea(x, y, r, minLevel, maxLevel);
    for (size_t i = 0; i < v.size() && (int)i < cap; i++) idx[i] = (int32_t)v[i];
    return (int)v.size();
}

// Frame::ComputeKeyPointRays + AssignFeaturesToGrid of GIVEN key points (scene::make_frame): rays, mGrid sizes, and the mGrid cell contents
// concatenated in (face, col, row) order. Every key point must lie on a face (ComputeKeyPointRays exits otherwise), and its cell corner on
// the same face (PosInGrid asserts otherwise).
void ref_frame_index(int n, const KpPOD* kps, float* rays, int32_t* gridCount, int32_t* cellIdx) {
    Frame* F = make_frame(n, kps, NULL, NULL);
    read_frame(*F, n, NULL, NULL, rays, gridCount);
    int m = 0;
    for (int f = 0; f < CUBEMAP_FACES; f++) for (int x = 0; x < CUBEFACE_GRID_COLS; x++) for (int y = 0; y < CUBEFACE_GRID_ROWS; y++)
        for (size_t j = 0; j < F->mGrid[f][x][y].size(); j++) cellIdx[m++] = (int32_t)F->mGrid[f][x][y][j];
    delete F;
}

// ---- projection matchers of the reference on objects built from flat arrays (what Tracking holds after Frame::Frame)
// ORBMatcher(0.9, checkOri).SearchByProjection(CurrentFrame, LastFrame, th, true)   src/ORBMatcher.cpp:130-251
int ref_search_by_projection_last(int nCur, const KpPOD* kCur, const uint8_t* dCur, const float* TcwCur, int nLast, const KpPOD* kLast, const float* TcwLast,
                                  const uint8_t* hasMP, const float* Xw, const uint8_t* dMP, const int32_t* mpObs, const uint8_t* curTaken, float th, int checkOri,
                                  int32_t* matchCur) {
    ProjectionLastScene s(nCur, kCur, dCur, TcwCur, nLast, kLast, TcwLast, hasMP, Xw, dMP, mpObs, curTaken);
    ORBMatcher matcher(0.9f, checkOri != 0);
    const int n = matcher.SearchByProjection(*s.cur, *s.last, th, true);
    s.read(matchCur);
    return n;
}

// ORBMatcher(nnratio).SearchByProjection(F, vpMapPoints, th)   src/ORBMatcher.cpp:51-128 ; the MapPoints carry what Frame::isInFrustum left in them
int ref_search_by_projection_local(int nF, const KpPOD* kF, const uint8_t* dF, int nMP, const uint8_t* inView, const float* projXY, const int32_t* level, const float* viewCos,
                                   const uint8_t* dMP, const int32_t* mpObs, const uint8_t* fTaken, float th, float nnratio, int32_t* matchF) {
    Map map;
    Frame* F = make_frame(nF, kF, dF, I4);
    std::vector<KpPOD> kd(nMP, kHolderKp);
    Frame* holder = make_frame(nMP, kd.data(), dMP, I4);   // only lends its descriptor rows to the MapPoint constructor
    KeyFrame* kfObs = new KeyFrame(*holder, &map, NULL);
    std::map<MapPoint*, int> idxOf; std::vector<MapPoint*> mps(nMP), owned;
    for (int m = 0; m < nMP; m++) {
        MapPoint* mp = new MapPoint(mat_from(P0, 3, 1), &map, holder, m);
        if (mpObs[m] > 0) mp->AddObservation(kfObs, m);
        mp->mbTrackInView = inView[m] != 0; mp->mTrackProjX = projXY[2 * m]; mp->mTrackProjY = projXY[2 * m + 1]; mp->mnTrackScaleLevel = level[m]; mp->mTrackViewCos = viewCos[m];
        mps[m] = mp; idxOf[mp] = m; owned.push_back(mp);
    }
    for (int i = 0; i < nF; i++) if (fTaken[i]) { MapPoint* mp = new MapPoint(mat_from(P0, 3, 1), kfObs, &map); mp->AddObservation(kfObs, 0); F->mvpMapPoints[i] = mp; idxOf[mp] = -2; owned.push_back(mp); }
    ORBMatcher matcher(nnratio, true);
    const int n = matcher.SearchByProjection(*F, mps, th);
    for (int i = 0; i < nF; i++) matchF[i] = F->mvpMapPoints[i] ? idxOf[F->mvpMapPoints[i]] : -1;
    for (MapPoint* mp : owned) delete mp;
    delete kfObs; delete F; delete holder;
    return n;
}
// CamModelGeneral::TransformRaysToCubemap(up, vp, x, y, z)
int ref_ray_to_cubemap(float x, float y, float z, float* up, float* vp) { return (int)CamModelGeneral::GetCamera()->TransformRaysToCubemap(*up, *vp, x, y, z); }

// the two matrix expressions every projection on the path goes through, evaluated by the cv:: shim (pinned against cv2.gemm in the tests):
// `Rcw*x3Dw+tcw` (src/ORBMatcher.cpp:161, src/Frame.cpp:205) and `-Rcw.t()*tcw` (src/ORBMatcher.cpp:144, src/Frame.cpp:194)
void ref_expr_Rx_plus_t(const float* R9, const float* x3, const float* t3, float* out3) {
    cv::Mat R(3, 3, CV_32F, (void*)R9), x(3, 1, CV_32F, (void*)x3), t(3, 1, CV_32F, (void*)t3);
    cv::Mat o = R * x + t;
    for (int i = 0; i < 3; i++) out3[i] = o.at<float>(i);
}
void ref_expr_neg_Rt_t(const float* R9, const float* t3, float* out3) {
    cv::Mat R(3, 3, CV_32F, (void*)R9), t(3, 1, CV_32F, (void*)t3);
    cv::Mat o = -R.t() * t;
    for (int i = 0; i < 3; i++) out3[i] = o.at<float>(i);
}

// timed CPU baseline (bench.py cpu_baseline.kind "reference"): warp + ORBextractor::operator() over nframes frames with nthreads independent
// workers, each owning its extractor like one reference process per core (Examples/cubemap_lafida.cpp:111). Per-frame outputs kps / desc:
// nframes x cap, for the extract+match baseline. Returns the total key point count.
long ref_warp_extract_batch_out(const uint8_t* fisheyes, int nframes, const float* map1, const float* map2, const uint8_t* mask, int nfeatures, float scaleFactor, int nlevels,
                                int iniTh, int minTh, int nthreads, int cap, cv::KeyPoint* kpsOut, uint8_t* descOut, int* nOut) {
    CamModelGeneral* cam = CamModelGeneral::GetCamera();
    const int W3 = cam->GetCubeFaceWidth() * 3, H3 = cam->GetCubeFaceHeight() * 3, Iw = cam->GetFisheyeWidth(), Ih = cam->GetFisheyeHeight();
    std::vector<long> totals(nthreads, 0);
    auto work = [&](int t) {
        ORBextractor ex(nfeatures, scaleFactor, nlevels, iniTh, minTh);
        cv::Mat canvas = cv::Mat::zeros(H3, W3, CV_8UC1), mk(H3, W3, CV_8UC1, (void*)mask), desc;
        cv::Mat m1(H3, W3, CV_32F, (void*)map1), m2(H3, W3, CV_32F, (void*)map2);
        std::vector<cv::KeyPoint> kps;
        for (int f = t; f < nframes; f += nthreads) {
            cv::Mat fe(Ih, Iw, CV_8UC1, (void*)(fisheyes + (size_t)f * Iw * Ih));
            warp_into(canvas, fe, m1, m2);
            ex(canvas, mk, kps, desc);
            const int m = std::min((int)kps.size(), cap);
            nOut[f] = m;
            if (m) std::memcpy((void*)(kpsOut + (size_t)f * cap), kps.data(), (size_t)m * sizeof(cv::KeyPoint));
            for (int i = 0; i < m; i++) std::memcpy(descOut + ((size_t)f * cap + i) * 32, desc.ptr<uchar>(i), 32);
            totals[t] += m;
        }
    };
    std::vector<std::thread> th;
    for (int t = 1; t < nthreads; t++) th.emplace_back(work, t);
    work(0);
    for (auto& x : th) x.join();
    long s = 0;
    for (long v : totals) s += v;
    return s;
}

// ---- DBoW2: ORBVocabulary (include/ORBVocabulary.h:35-36) loaded from a text file like System does (src/System.cpp:52-61), transform like Frame::ComputeBoW
void* ref_voc_load(const char* path) {
    ORBVocabulary* v = new ORBVocabulary();
    if (!v->loadFromTextFile(path)) { delete v; return nullptr; }
    return v;
}
void ref_voc_destroy(void* v) { delete (ORBVocabulary*)v; }
int ref_voc_size(void* v) { return (int)((ORBVocabulary*)v)->size(); }
// bowWord / bowVal: the BowVector in map order; nodeOf[i]: FeatureVector node of feature i (-1 if the feature is in no node list)
int ref_voc_transform(void* vv, const uint8_t* feats, int n, int levelsup, int32_t* bowWord, double* bowVal, int32_t* nodeOf) {
    ORBVocabulary* voc = (ORBVocabulary*)vv;
    cv::Mat D(n, 32, CV_8UC1, (void*)feats);
    std::vector<cv::Mat> vCurrentDesc = Converter::toDescriptorVector(D);   // src/Frame.cpp:723
    DBoW2::BowVector bv; DBoW2::FeatureVector fv;
    voc->transform(vCurrentDesc, bv, fv, levelsup);
    int m = 0;
    for (DBoW2::BowVector::const_iterator it = bv.begin(); it != bv.end(); ++it, ++m) { bowWord[m] = (int32_t)it->first; bowVal[m] = it->second; }
    for (int i = 0; i < n; i++) nodeOf[i] = -1;
    for (DBoW2::FeatureVector::const_iterator it = fv.begin(); it != fv.end(); ++it)
        for (size_t k = 0; k < it->second.size(); k++) nodeOf[it->second[k]] = (int32_t)it->first;
    return m;
}

// ORBMatcher::DescriptorDistance, src/ORBMatcher.cpp:951-967
int ref_descriptor_distance(const uint8_t* a, const uint8_t* b) {
    cv::Mat ma(1, 32, CV_8UC1, (void*)a), mb(1, 32, CV_8UC1, (void*)b);
    return ORBMatcher::DescriptorDistance(ma, mb);
}

// =========================================================================================== LocalMapping feature operations (SURVEY §8(f) rank 4)
// MapPoint::ComputeDistinctiveDescriptors on a MapPoint observed once in each of N key frames (observation i carries desc row i); out = mDescriptor
void ref_distinctive_descriptor(int N, const uint8_t* desc, uint8_t* out32) {
    const int32_t offset[2] = {0, N};
    DistinctiveScene s(1, offset, desc);
    s.mps[0]->ComputeDistinctiveDescriptors();
    std::memcpy(out32, s.mps[0]->GetDescriptor().ptr<uchar>(0), 32);
}

// ORBMatcher(0.6).Fuse(pKF, vpMapPoints, th) on the scene of FuseScene. Outputs: valid / level = the pre-tests and PredictScale of Fuse evaluated
// with the reference's own getters; idxInKF[m] = FuseScene::index_in_kf after the call. Returns nFused.
int ref_fuse(int nKF, const KpPOD* kKF, const uint8_t* dKF, const float* Tcw, int nMP, const float* Xw, const KpPOD* kObs, const uint8_t* dMP, const float* TcwObs, float th,
             uint8_t* valid, int32_t* level, int32_t* idxInKF) {
    FuseScene s(nKF, kKF, dKF, Tcw, nMP, Xw, kObs, dMP, TcwObs);
    cv::Mat Ow = s.pKF->GetCameraCenter();
    for (int m = 0; m < nMP; m++) {   // src/ORBMatcher.cpp:1145-1178 with the reference's own accessors
        MapPoint* pMP = s.mps[m];
        valid[m] = 0; level[m] = 0;
        cv::Mat p3Dw = pMP->GetWorldPos();
        const float maxDistance = pMP->GetMaxDistanceInvariance();
        const float minDistance = pMP->GetMinDistanceInvariance();
        cv::Mat PO = p3Dw - Ow;
        const float dist3D = cv::norm(PO);
        if (dist3D < minDistance || dist3D > maxDistance) continue;
        cv::Mat Pn = pMP->GetNormal();
        if (PO.dot(Pn) < 0.5 * dist3D) continue;
        valid[m] = 1; level[m] = pMP->PredictScale(dist3D, s.pKF);
    }
    ORBMatcher matcher(0.6f, true);
    const int nFused = matcher.Fuse(s.pKF, s.mps, th);
    for (int m = 0; m < nMP; m++) idxInKF[m] = s.index_in_kf(m);
    return nFused;
}

// ORBMatcher(0.6, checkOri).SearchForTriangulation(pKF1, pKF2, E12, pairs) on the scene of TriangulationScene. Ow1out = pKF1->GetCameraCenter().
// match12[i1] = i2 or -1. Returns nmatches.
int ref_search_for_triangulation(int n1, const KpPOD* k1, const uint8_t* d1, const float* Tcw1, const uint8_t* hasMP1, const int32_t* node1, int n2, const KpPOD* k2,
                                 const uint8_t* d2, const float* Tcw2, const uint8_t* hasMP2, const int32_t* node2, const float* E12, int checkOri, float* Ow1out,
                                 int32_t* match12) {
    TriangulationScene s(n1, k1, d1, Tcw1, hasMP1, node1, n2, k2, d2, Tcw2, hasMP2, node2);
    cv::Mat Ow = s.kf1->GetCameraCenter();
    for (int i = 0; i < 3; i++) Ow1out[i] = Ow.at<float>(i);
    ORBMatcher matcher(0.6f, checkOri != 0);
    std::vector<std::pair<size_t, size_t> > pairs;
    const int n = matcher.SearchForTriangulation(s.kf1, s.kf2, mat_from(E12, 3, 3), pairs);
    s.read(pairs, match12);
    return n;
}

// CamModelGeneral::GetVectorSigma(key, normalRig)
float ref_vector_sigma(float kx, float ky, const float* normalRig) {
    cv::KeyPoint kp; kp.pt.x = kx; kp.pt.y = ky;
    return CamModelGeneral::GetCamera()->GetVectorSigma(kp, cv::Vec3f(normalRig[0], normalRig[1], normalRig[2]));
}

}  // extern "C"
