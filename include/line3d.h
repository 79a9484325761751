/* include/line3d.h — L3DPP::Line3D on the GPU: the host-side mirror of the reference's public class (line3D.h:61-233).
 *
 * Same class name, method names, argument meaning, defaults and output types (FinalLine3D / LineCluster3D /
 * Segment3D / Segment2D, segment3D.h:35-178, commons.h:103-133) so an SfM frontend written against the reference
 * (main_vsfm.cpp:306-330 etc.) ports by recompiling.  Everything data-parallel goes through the C ABI of
 * include/l3d_capi.h; this class only does what line3D.cc does on the host around the accelerator calls.
 *
 * Differences forced by this image (no Eigen / OpenCV / Boost headers):
 *   - Matrix3d / Vector3d / Vec4f are small PODs.  When <eigen3/Eigen/Eigen> and <opencv2/core.hpp> are on the include path
 *     (or L3DPP_WITH_EIGEN_OPENCV is defined) the reference's own addImage signature (line3D.h:104-108: cv::Mat&,
 *     Eigen::Matrix3d, Eigen::Vector3d, std::vector<cv::Vec4f>) is available as an inline overload that converts and
 *     forwards; tests/test_cpu.py compiles it against the header stand-ins of oracle/ref_shim.  get3Dlines() returns the POD
 *     types (P1().x is a member, not Eigen's x()): a frontend that reads the result lines needs that one-character change.
 *   - addImage takes the image (an Image8u, or its size alone) and the 2D segments (the reference's own line_segments argument,
 *     line3D.h:102-108).  With no segments it reads the reference's segment cache
 *     <output_folder>/L3D++_data/segments_L3D++_<camID>_<w>x<h>_3000.bin (line3D.cc:295-309; segmentCachePath in include/line3d_io.h)
 *     when load_segments is true and the file exists, so a folder the reference has run on gives it exactly the segments the reference
 *     used.  Otherwise the image overload does what the reference's detectLineSegments (line3D.cc:249-372) does around its LSD call:
 *     grey conversion and the max_img_width resize on the GPU (l3d_prepare_gray_u8, bit-exact to OpenCV), then the detector the
 *     caller registered with setSegmentDetector, then the upscale, length filter, longest-first order and max_line_segments cut, and
 *     the segment cache is written.  The detector itself (LSD) is outside this library (SURVEY.md §2 row 13): without one, and without
 *     segments or a cache file, the view is rejected and lastError() names the file that was looked for.
 *   - undistortImage (line3D.h:119-122) takes the owning Image8u and the POD vectors; with Eigen / OpenCV headers the reference's
 *     cv::Mat signature is an inline overload for CV_8UC1 / CV_8UC3.  It runs on the GPU and its map is defined by an explicit
 *     formula, which OpenCV builds reproduce to within one 1/32-px step (DESIGN.md §4a).
 *   - save3DLinesAsBIN writes the reference's Boost binary archive without Boost (csrc/line3d_bin.cc, DESIGN.md §6a), like the
 *     TXT / OBJ / STL writers; read3DLinesBIN reads such files back.
 *   - use_GPU selects the SCORING SEMANTICS of the reference's two paths; both run on the GPU (there is no CPU path).
 */
#ifndef L3DPP_B200_LINE3D_H_
#define L3DPP_B200_LINE3D_H_

#include <cstddef>
#include <cstring>
#include <list>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#if !defined(L3DPP_WITH_EIGEN_OPENCV) && defined(__has_include)
#if __has_include(<eigen3/Eigen/Eigen>) && __has_include(<opencv2/core.hpp>)
#define L3DPP_WITH_EIGEN_OPENCV 1
#endif
#endif
#ifdef L3DPP_WITH_EIGEN_OPENCV
#include <eigen3/Eigen/Eigen>
#include <opencv2/core.hpp>
#endif

namespace L3DPP {

struct Vector2d { double x, y; Vector2d() : x(0), y(0) {} Vector2d(double a, double b) : x(a), y(b) {} };
struct Vector3d { double x, y, z; Vector3d() : x(0), y(0), z(0) {} Vector3d(double a, double b, double c) : x(a), y(b), z(c) {} };
struct Matrix3d { double m[9]; double& operator()(int r, int c) { return m[r * 3 + c]; } double operator()(int r, int c) const { return m[r * 3 + c]; } };
struct Vec4f { float v[4]; float operator()(int i) const { return v[i]; } };
struct Vector4f { float v[4]; float operator()(int i) const { return v[i]; } };

/* an 8-bit image that owns its pixels: rows x cols, 1 or 3 interleaved channels, rows packed (the layout of a continuous CV_8UC1 /
 * CV_8UC3 cv::Mat) */
struct Image8u {
    int cols, rows, channels;
    std::vector<unsigned char> data;
    Image8u() : cols(0), rows(0), channels(1) {}
    Image8u(int r, int c, int ch) : cols(c), rows(r), channels(ch), data((size_t)(r > 0 ? r : 0) * (c > 0 ? c : 0) * (ch > 0 ? ch : 0)) {}
};

/* a camera's lens distortion as OpenCV models it (include/l3d_capi.h l3d_undistort_desc).  RADTAN: k = k1..k6 (OpenCV's
 * (k1, k2, p1, p2, k3, k4, k5, k6); k4..k6 = 0 is the 5-coefficient model), p = p1, p2.  FISHEYE: cv::fisheye's k1..k4 in k[0..3],
 * the rest zero.  Zero-initialised: no distortion. */
struct LensDistortion {
    enum Model { RADTAN = 0, FISHEYE = 1 };
    int model;
    double k[6], p[2];
};

#ifdef L3DPP_WITH_EIGEN_OPENCV
namespace detail {
/* the pixels of a cv::Mat as an Image8u, honouring its row step; a type other than CV_8UC1 / CV_8UC3 gives 0 channels, which
 * addImage rejects as the reference does (line3D.cc:251-266) */
template <class M>
auto imageOf(const M& m, int) -> decltype((void)m.data, (void)m.step, Image8u())
{
    const bool ok = m.type() == CV_8UC1 || m.type() == CV_8UC3;
    Image8u img(m.rows, m.cols, ok ? m.channels() : 0);
    const size_t row = (size_t)m.cols * img.channels, step = static_cast<size_t>(m.step);
    for (int r = 0; r < m.rows && row; ++r) std::memcpy(img.data.data() + r * row, m.data + r * step, row);
    return img;
}
/* a cv::Mat stand-in that carries no pixels (the header stand-ins of the verbatim reference build) gives its size and no pixels:
 * addImage can still use the segment cache, and rejects the view if it would have to prepare the image */
template <class M>
Image8u imageOf(const M& m, long)
{
    Image8u img;
    img.rows = m.rows; img.cols = m.cols; img.channels = m.channels();
    return img;
}
}  // namespace detail
#endif

/* defaults: commons.h:41-69 */
const int L3D_DEF_MAX_IMG_WIDTH = -1;
const unsigned int L3D_DEF_MAX_NUM_SEGMENTS = 3000;
const bool L3D_DEF_LOAD_AND_STORE_SEGMENTS = true;
const float L3D_DEF_COLLINEARITY_T = -1.0f;
const unsigned int L3D_DEF_MATCHING_NEIGHBORS = 10;
const float L3D_DEF_EPIPOLAR_OVERLAP = 0.25f;
const int L3D_DEF_KNN = 10;
const float L3D_DEF_SCORING_POS_REGULARIZER = 2.5f;
const float L3D_DEF_SCORING_ANG_REGULARIZER = 10.0f;
const bool L3D_DEF_PERFORM_RDD = false;
const unsigned int L3D_DEF_MIN_VISIBILITY_T = 3;
const bool L3D_DEF_USE_CERES = false;
const unsigned int L3D_DEF_CERES_MAX_ITER = 250;

class Segment2D {   /* commons.h:103-133 */
public:
    Segment2D() : camID_(0), segID_(0) {}
    Segment2D(unsigned int camID, unsigned int segID) : camID_(camID), segID_(segID) {}
    unsigned int camID() const { return camID_; }
    unsigned int segID() const { return segID_; }
    bool operator==(const Segment2D& r) const { return camID_ == r.camID_ && segID_ == r.segID_; }
    bool operator<(const Segment2D& r) const { return camID_ < r.camID_ || (camID_ == r.camID_ && segID_ < r.segID_); }
    bool operator!=(const Segment2D& r) const { return !(*this == r); }
private:
    unsigned int camID_, segID_;
};

class Segment3D {   /* segment3D.h:35-94 */
public:
    Segment3D();
    Segment3D(const Vector3d& P1, const Vector3d& P2);
    /* every stored field as given, nothing recomputed: how a segment read from a .bin file (read3DLinesBIN) keeps its bits */
    Segment3D(const Vector3d& P1, const Vector3d& P2, const Vector3d& dir, float length, bool valid)
        : P1_(P1), P2_(P2), dir_(dir), length_(length), valid_(valid) {}
    float distance_Point2Line(const Vector3d& P) const;
    void translate(const Vector3d& t);
    Vector3d P1() const { return P1_; }
    Vector3d P2() const { return P2_; }
    Vector3d dir() const { return dir_; }
    float length() const { return length_; }
    bool valid() const { return valid_; }
private:
    Vector3d P1_, P2_, dir_;
    float length_;
    bool valid_;
};

class LineCluster3D {   /* segment3D.h:124-151 */
public:
    LineCluster3D() : reference_view_(0) {}
    LineCluster3D(const Segment3D& seg3D, const std::list<Segment2D>& residuals, unsigned int ref_view)
        : seg3D_(seg3D), residuals_(residuals), reference_view_(ref_view) {}
    Segment3D seg3D() const { return seg3D_; }
    const std::list<Segment2D>* residuals() const { return &residuals_; }
    size_t size() const { return residuals_.size(); }
    unsigned int reference_view() const { return reference_view_; }
    void update3Dline(const Segment3D& s) { seg3D_ = s; }
    void translate(const Vector3d& t) { seg3D_.translate(t); }
private:
    Segment3D seg3D_;
    std::list<Segment2D> residuals_;
    unsigned int reference_view_;
};

struct FinalLine3D {   /* segment3D.h:155-163 */
    std::list<Segment3D> collinear3Dsegments_;
    LineCluster3D underlyingCluster_;
};

/* counters the reference prints to stdout (SURVEY.md §5 "Metrics / logging"); handy parity checkpoints.  pair_evaluations: the
 * (source, target) cells matchImages evaluated, Ns*Nt per scanned view pair and the distinct listed correspondences of a pair
 * restricted by setLineCandidates */
struct Line3DStats {
    long long view_pairs, pair_evaluations, matches_after_knn, estimates, affinity_entries, affinity_rows, clusters_total,
        clusters_valid, lines3D, collinear_entries, opt_iterations;
    double ms_match, ms_score, ms_affinity, ms_diffusion, ms_cluster, opt_cost_before, opt_cost_after;
    double ms_gather;      /* the part of ms_match that gathered the other devices' rows on the first one (device time); 0 on one device */
};

class Line3D {
public:
    /* line3D.h:80-85.  output_folder / load_segments / max_img_width / max_line_segments only matter for addImage without segments
     * (segment cache, image preparation, the cut of the detections) and the output filename (createOutputFilename). */
    Line3D(const std::string& output_folder, const bool load_segments = L3D_DEF_LOAD_AND_STORE_SEGMENTS,
           const int max_img_width = L3D_DEF_MAX_IMG_WIDTH, const unsigned int max_line_segments = L3D_DEF_MAX_NUM_SEGMENTS,
           const bool neighbors_by_worldpoints = true, const bool use_GPU = true, const int cuda_device = 0);
    /* The same on several GPUs (an addition): cuda_devices[0] is the primary, where the scoring sweep, affinity, diffusion, clustering
     * and bundling run and where the results live.  matchImages splits the view pairs over all listed devices by cost (Ns * Nt), matches
     * every share from its own host thread and gathers the rows on the primary (l3d_match_gather), so the results, stats included, are
     * those of one device bit for bit.  A device may be listed more than once (several contexts on one GPU).  Every device holds all
     * segments and the count / record arrays of the whole job (DESIGN.md §5).  Throws std::invalid_argument for an empty list and
     * std::runtime_error if a device cannot be used.  The constructor above means {cuda_device}. */
    Line3D(const std::string& output_folder, const bool load_segments, const int max_img_width, const unsigned int max_line_segments,
           const bool neighbors_by_worldpoints, const bool use_GPU, const std::vector<int>& cuda_devices);
    ~Line3D();
    Line3D(const Line3D&) = delete;
    Line3D& operator=(const Line3D&) = delete;

    /* line3D.h:104-108 with (image_width, image_height) instead of cv::Mat& image.  An empty line_segments list reads the segment
     * cache segmentCachePath(output_folder, camID, image_width, image_height, max_img_width) when load_segments is true; its
     * segments are used as stored (line3D.cc:303-307: already upscaled, length-filtered and longest first, not truncated). */
    /* Returns false (and sets lastError(), which a later successful addImage does not clear) if the view was rejected. */
    bool addImage(const unsigned int camID, const int image_width, const int image_height, const Matrix3d& K, const Matrix3d& R,
                  const Vector3d& t, const float median_depth, const std::list<unsigned int>& wps_or_neighbors,
                  const std::vector<Vec4f>& line_segments);

    /* line3D.h:104-108 with an Image8u (1 or 3 channels, channel 0 is R).  In the reference's order (line3D.cc:116-186, 249-372): the
     * size check and the camera-ID check (an ID is reserved while its image is prepared, so a repeated ID never reaches the detector)
     * come first.  Given segments are used as they are.  Otherwise the segment cache is read as above; on a miss the image is
     * prepared on the GPU (grey, and resized when its larger side exceeds max_img_width: l3d_prepare_gray_u8), handed to the
     * setSegmentDetector function, and its detections are scaled back to the image's size, kept when longer than
     * 0.005 * the image diagonal, ordered longest first by the reference's std::priority_queue and cut at max_line_segments; when
     * load_segments is true and a segment survives, they are written to the segment cache (the L3D++_data folder is created if
     * needed; a cache that cannot be written is only reported in verbose mode, the view is still added).  Rejected with lastError() set: no detector and no cache file (the message names the file), a detector that returns
     * false, no detection longer than the threshold, an image that is not 8-bit grey or RGB.  Thread-safe: the GPU step of concurrent
     * calls is serialised on the primary device; the detector runs on the calling thread outside every lock. */
    bool addImage(const unsigned int camID, const Image8u& image, const Matrix3d& K, const Matrix3d& R, const Vector3d& t,
                  const float median_depth, const std::list<unsigned int>& wps_or_neighbors,
                  const std::vector<Vec4f>& line_segments = std::vector<Vec4f>());

    /* addImage for a camera with lens distortion (an addition): `image` and `line_segments` are in the DISTORTED image; the view is
     * added as the undistorted camera K.  Given segments: their endpoints go through undistortPoints(lens, K) (in pixels of K), then as
     * above.  No segments: the segment cache is read as above and its segments are used as stored (the cache holds detections in the
     * undistorted image).  On a miss the image is undistorted into K and prepared on the GPU without leaving the device in between
     * (l3d_undistort_u8 then l3d_prepare_gray_u8), and only the prepared image comes back for the detector: the segments, the cache
     * written and the detector's input are byte for byte those of undistortImage(image, u, lens, K) followed by addImage(u).  An all-zero
     * lens is the overload above.  A camera or lens l3d_undistort_u8 rejects rejects the view (lastError() set). */
    bool addImage(const unsigned int camID, const Image8u& image, const Matrix3d& K, const Matrix3d& R, const Vector3d& t,
                  const float median_depth, const std::list<unsigned int>& wps_or_neighbors, const LensDistortion& lens,
                  const std::vector<Vec4f>& line_segments = std::vector<Vec4f>());
    /* the (image_width, image_height) form: given segments are undistorted as above; an empty list reads the segment cache as stored */
    bool addImage(const unsigned int camID, const int image_width, const int image_height, const Matrix3d& K, const Matrix3d& R,
                  const Vector3d& t, const float median_depth, const std::list<unsigned int>& wps_or_neighbors, const LensDistortion& lens,
                  const std::vector<Vec4f>& line_segments);

#ifdef L3DPP_WITH_EIGEN_OPENCV
    /* The reference's exact signature (line3D.h:104-108) for CV_8UC1 / CV_8UC3 images of any row step: the image overload above.
     * With segments given only the image's size is used.  A template only so that this header also compiles against cv::Mat
     * stand-ins that carry no pixels; calls are written as for the reference. */
    template <class MatT = cv::Mat>
    bool addImage(const unsigned int camID, cv::Mat& image, const Eigen::Matrix3d& K, const Eigen::Matrix3d& R, const Eigen::Vector3d& t,
                  const float median_depth, const std::list<unsigned int>& wps_or_neighbors,
                  const std::vector<cv::Vec4f>& line_segments = std::vector<cv::Vec4f>())
    {
        Matrix3d Kp, Rp;
        for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) { Kp(r, c) = K(r, c); Rp(r, c) = R(r, c); }
        std::vector<Vec4f> segs(line_segments.size());
        for (size_t i = 0; i < line_segments.size(); ++i) for (int k = 0; k < 4; ++k) segs[i].v[k] = line_segments[i](k);
        const Vector3d tp(t(0), t(1), t(2));
        const MatT& img = image;
        if (!segs.empty()) return addImage(camID, img.cols, img.rows, Kp, Rp, tp, median_depth, wps_or_neighbors, segs);
        return addImage(camID, detail::imageOf(img, 0), Kp, Rp, tp, median_depth, wps_or_neighbors, segs);
    }
#endif

    /* The line detector addImage calls on the prepared grey image (what the reference does with
     * cv::createLineSegmentDetector(cv::LSD_REFINE_ADV)->detect, line3D.cc:311-317): fill `detections` with (x1, y1, x2, y2) in the
     * coordinates of `gray` and return true, or return false to reject the view.  Called from the thread that called addImage, with
     * no lock held: concurrent addImage calls run it concurrently, so it must be thread-safe.  nullptr: no detector. */
    typedef bool (*SegmentDetectorFn)(void* user, const Image8u& gray, std::vector<Vec4f>& detections);
    void setSegmentDetector(SegmentDetectorFn detector, void* user);

    /* Restrict the matching of the view pair {camA, camB} to the given correspondences (segment of camA, segment of camB), e.g. from a
     * descriptor or learned line matcher, line tracking or an SfM tool.  For each source segment of a restricted pair matchImages
     * evaluates only the listed target segments, with everything else as the epipolar scan does it: the exact arithmetic of the
     * semantics, the epipolar_overlap and depth tests, the kNN rule (kNN <= 0: all, ascending target; kNN > 32: all, then the cut) and
     * the tie order (overlap descending, then the smaller target segment).  Listing every target segment of a pair gives the scan's
     * matches.  An empty list restricts the pair to no matches.  Either camera order, duplicates allowed; a second call for the same
     * pair replaces its list; the lists stay until clearLineCandidates().  Pairs without a list are scanned as before, and the visual
     * neighbours are chosen as before: a list of a pair matchImages does not evaluate (not neighbours, or a camera never added) is
     * ignored (verbose mode reports how many).  camA == camB is rejected with lastError() set; a segment ID at or beyond its view's
     * segment count makes matchImages fail, naming the camera and segment.  stats().pair_evaluations counts Ns*Nt for a scanned pair
     * and the distinct listed correspondences for a restricted one. */
    void setLineCandidates(const unsigned int camA, const unsigned int camB, const std::vector<std::pair<unsigned int, unsigned int> >& seg_pairs);
    void clearLineCandidates();

    /* line3D.h:140-145.  kNN in 1..32: the kNN best matches of every segment.  kNN <= 0 (keep all) or kNN > 32 (keep all, then cut
     * every segment to its kNN best): a segment may have at most 8533 matches in one view pair before the cut (the rows are sorted in
     * 200 KiB of shared memory, 24 B per match); more makes matchImages fail with lastError() naming the limit, where the reference has none. */
    void matchImages(const float sigma_position = L3D_DEF_SCORING_POS_REGULARIZER, const float sigma_angle = L3D_DEF_SCORING_ANG_REGULARIZER,
                     const unsigned int num_neighbors = L3D_DEF_MATCHING_NEIGHBORS, const float epipolar_overlap = L3D_DEF_EPIPOLAR_OVERLAP,
                     const int kNN = L3D_DEF_KNN, const float const_regularization_depth = -1.0f);

    /* line3D.h:162-166.  use_CERES: the bundling of optimization.cc runs on the GPU (l3d_optimize_lines); Ceres is not needed,
     * so the flag is honoured in every build (the reference silently drops it when it was built without Ceres, line3D.cc:1738-1744) */
    void reconstruct3Dlines(const unsigned int visibility_t = L3D_DEF_MIN_VISIBILITY_T, const bool perform_diffusion = L3D_DEF_PERFORM_RDD,
                            const float collinearity_t = L3D_DEF_COLLINEARITY_T, const bool use_CERES = L3D_DEF_USE_CERES,
                            const unsigned int max_iter_CERES = L3D_DEF_CERES_MAX_ITER);

    void get3Dlines(std::vector<FinalLine3D>& result);                 /* line3D.h:173 */
    void saveResultAsSTL(const std::string& output_folder);            /* line3D.h:183-185 */
    void saveResultAsOBJ(const std::string& output_folder);
    void save3DLinesAsTXT(const std::string& output_folder);
    /* line3D.h:185: <output_folder>/<createOutputFilename()>.bin, the reference's Boost binary archive of get3Dlines() (every
     * field at full precision; read it back with read3DLinesBIN, include/line3d_io.h).  With no 3D lines nothing is written. */
    void save3DLinesAsBIN(const std::string& output_folder);
    Vector4f getSegmentCoords2D(const Segment2D& seg2D);               /* line3D.h:196-198 */
    Vector4f getSegmentCoords2D(const unsigned int camID, const unsigned int segID);
    size_t numImages();                                                /* line3D.h:205 */
    std::string createOutputFilename();                                /* line3D.h:224 */
    static Matrix3d rotationFromQ(const double Qw, const double Qx, const double Qy, const double Qz);   /* line3D.h:219-220 */
    /* line3D.cc:2714-2727: Rz(yaw) * Ry(pitch) * Rx(roll), each as Eigen's AngleAxisd(angle, unit axis).toRotationMatrix() forms it
     * (the mavmap frontend's camera rotation).  Returns the POD Matrix3d, like rotationFromQ. */
    static Matrix3d rotationFromRPY(const double roll, const double pitch, const double yaw);
    /* line3D.cc:2784-2852: K, R, t with P = K [R|t] (P: 3x4, row-major) by the reference's RQ decomposition: Givens rotations
     * Rx, Ry, Rz on P's left 3x3 block, the column-sign fix (positive diagonal of K), R = (Rx Ry Rz Sign)^T, t = K^-1 P4 with K
     * before normalisation, then K divided by K(2,2). */
    static void decomposeProjectionMatrix(const double P[12], Matrix3d& K, Matrix3d& R, Vector3d& t);
#ifdef L3DPP_WITH_EIGEN_OPENCV
    /* the reference's signature (line3D.h:230-233); a P that is not 3x4 leaves the outputs untouched (the reference prints a message) */
    static void decomposeProjectionMatrix(const Eigen::MatrixXd P_in, Eigen::Matrix3d& K_out, Eigen::Matrix3d& R_out, Eigen::Vector3d& t_out)
    {
        if (P_in.rows() != 3 || P_in.cols() != 4) return;
        double P[12];
        for (int r = 0; r < 3; ++r) for (int c = 0; c < 4; ++c) P[4 * r + c] = P_in(r, c);
        Matrix3d K, R; Vector3d t;
        decomposeProjectionMatrix(P, K, R, t);
        for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) { K_out(r, c) = K(r, c); R_out(r, c) = R(r, c); }
        t_out(0) = t.x; t_out(1) = t.y; t_out(2) = t.z;
    }
#endif

    /* line3D.h:119-122: lens undistortion as the reference does it with OpenCV (initUndistortRectifyMap with fixed-point maps +
     * remap, bilinear, border 0; include/l3d_capi.h l3d_undistort_u8).  Uses K(0,0), K(1,1), K(0,2), K(1,2) only; out gets the size
     * and channels of in (in == out is allowed).  Runs on the calling thread's current CUDA device through a context that lives for
     * the call.  Throws std::invalid_argument for an image or camera l3d_undistort_u8 rejects, std::runtime_error on a CUDA failure
     * or without a usable device. */
    static void undistortImage(const Image8u& in, Image8u& out, const Vector3d& radial_coeffs, const Vector2d& tangential_coeffs, const Matrix3d& K);
    /* the same for any lens l3d_undistort_u8 takes (the overload above is lens = {RADTAN, {k1, k2, k3, 0, 0, 0}, {p1, p2}});
     * std::invalid_argument also for an unknown model and a fisheye lens with k[4], k[5], p[0] or p[1] nonzero */
    static void undistortImage(const Image8u& in, Image8u& out, const LensDistortion& lens, const Matrix3d& K);
    /* the same into a chosen camera matrix and size: OpenCV's initUndistortRectifyMap(K, D, I, newK, Size(out_width, out_height)) (or
     * cv::fisheye's with P = newK) + remap.  Uses newK(0,0), newK(1,1), newK(0,2), newK(1,2); those four all zero: K.  out_width and
     * out_height both 0: the size of in; out gets out_height x out_width and the channels of in.  With newK zero and the size 0 (or
     * newK = K and the size of in) this is the overload above, byte for byte.  std::invalid_argument also for a new K or size
     * l3d_undistort_u8 rejects (include/l3d_capi.h). */
    static void undistortImage(const Image8u& in, Image8u& out, const LensDistortion& lens, const Matrix3d& K, const Matrix3d& newK, int out_width,
                               int out_height);
    /* cv::getOptimalNewCameraMatrix(K, D, Size(width, height), alpha, Size(new_width, new_height), validPixROI, centerPrincipalPoint) for
     * a RADTAN lens (5 or 8 coefficients), restated in double on the host as OpenCV 4.13 computes it (DESIGN.md §4a).  new_width /
     * new_height 0: the image size.  validPixROI (optional): x, y, width, height of the all-valid pixels in the new image.  Skew is
     * taken as zero.  std::invalid_argument for a fisheye lens, a size below 1, or fx / fy zero or not finite. */
    static Matrix3d getOptimalNewCameraMatrix(const Matrix3d& K, const LensDistortion& lens, int width, int height, double alpha, int new_width = 0,
                                              int new_height = 0, int validPixROI[4] = nullptr, bool centerPrincipalPoint = false);
    /* cv::fisheye::estimateNewCameraMatrixForUndistortRectify(K, D, Size(width, height), I, P, balance, Size(new_width, new_height),
     * fov_scale) for a FISHEYE lens, restated in double on the host (DESIGN.md §4a); R is the identity.  Same exceptions, for a
     * radtan lens instead. */
    static Matrix3d estimateNewCameraMatrixForUndistortRectify(const Matrix3d& K, const LensDistortion& lens, int width, int height, double balance = 0.0,
                                                               int new_width = 0, int new_height = 0, double fov_scale = 1.0);

    /* Lens undistortion of points (an addition): cv::undistortPoints(xy, xy, K, D, noArray(), newK) for a RADTAN lens and
     * cv::fisheye::undistortPoints(xy, xy, K, D, I, newK) for a FISHEYE lens, in place on interleaved x, y float pairs, on the GPU
     * (include/l3d_capi.h l3d_undistort_points; DESIGN.md §4a).  The result is in pixels of newK; newK all zero (the default): K.  Uses
     * K(0,0), K(1,1), K(0,2), K(1,2) and the same four entries of newK.  Runs on the calling thread's current CUDA device through a context
     * that lives for the call.  Throws std::invalid_argument for an odd number of coordinates and for a camera, lens or new K
     * l3d_undistort_points rejects, std::runtime_error on a CUDA failure or without a usable device. */
    static void undistortPoints(std::vector<float>& xy, const LensDistortion& lens, const Matrix3d& K, const Matrix3d& newK = Matrix3d());
    /* the same for both endpoints of every segment (x1, y1, x2, y2): what a segment detected in the distorted image is in the
     * undistorted one, endpoints only */
    static void undistortSegments(std::vector<Vec4f>& segs, const LensDistortion& lens, const Matrix3d& K, const Matrix3d& newK = Matrix3d());
    /* many point sets, each with its own lens, K and new K, in one launch: xy[i] with lenses[i], K[i] and newK[i] (newK empty: every set
     * into its K).  Same exceptions, and std::invalid_argument when the lists differ in length. */
    static void undistortPoints(std::vector<std::vector<float> >& xy, const std::vector<LensDistortion>& lenses, const std::vector<Matrix3d>& K,
                                const std::vector<Matrix3d>& newK = std::vector<Matrix3d>());
#ifdef L3DPP_WITH_EIGEN_OPENCV
    /* undistortSegments for cv::Vec4f segments (e.g. from cv::LineSegmentDetector or a segment file read into them) */
    template <class MatT = cv::Mat>
    static void undistortSegments(std::vector<cv::Vec4f>& segs, const LensDistortion& lens, const Eigen::Matrix3d& K,
                                  const Eigen::Matrix3d& newK = Eigen::Matrix3d::Zero())
    {
        std::vector<Vec4f> s(segs.size());
        for (size_t i = 0; i < segs.size(); ++i) for (int k = 0; k < 4; ++k) s[i].v[k] = segs[i](k);
        Matrix3d Kp, nKp;
        for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) { Kp(r, c) = K(r, c); nKp(r, c) = newK(r, c); }
        undistortSegments(s, lens, Kp, nKp);
        for (size_t i = 0; i < segs.size(); ++i) for (int k = 0; k < 4; ++k) segs[i](k) = s[i].v[k];
    }
#endif

#ifdef L3DPP_WITH_EIGEN_OPENCV
    /* The reference's exact signature for CV_8UC1 / CV_8UC3 images; honours the row step of inImg and create()s outImg.  A template
     * only so that this header also compiles against cv::Mat stand-ins that carry no pixels; calls are written as for the reference. */
    template <class MatT = cv::Mat>
    static void undistortImage(const cv::Mat& inImg, cv::Mat& outImg, const Eigen::Vector3d& radial_coeffs, const Eigen::Vector2d& tangential_coeffs,
                               const Eigen::Matrix3d& K)
    {
        const MatT& in = inImg;
        MatT& out = outImg;
        if (in.type() != CV_8UC1 && in.type() != CV_8UC3) throw std::invalid_argument("undistortImage: only CV_8UC1 and CV_8UC3 images");
        Image8u a(in.rows, in.cols, in.channels()), b;
        const size_t row = (size_t)in.cols * in.channels(), in_step = static_cast<size_t>(in.step);
        for (int r = 0; r < in.rows; ++r) std::memcpy(a.data.data() + r * row, in.data + r * in_step, row);
        Matrix3d Kp;
        for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) Kp(r, c) = K(r, c);
        undistortImage(a, b, Vector3d(radial_coeffs(0), radial_coeffs(1), radial_coeffs(2)), Vector2d(tangential_coeffs(0), tangential_coeffs(1)), Kp);
        out.create(in.rows, in.cols, in.type());
        const size_t out_step = static_cast<size_t>(out.step);
        for (int r = 0; r < b.rows; ++r) std::memcpy(out.data + r * out_step, b.data.data() + r * row, row);
    }
    /* the cv::Mat form of the LensDistortion overload (e.g. with readColmap's lenses) */
    template <class MatT = cv::Mat>
    static void undistortImage(const cv::Mat& inImg, cv::Mat& outImg, const LensDistortion& lens, const Eigen::Matrix3d& K)
    {
        const MatT& in = inImg;
        MatT& out = outImg;
        if (in.type() != CV_8UC1 && in.type() != CV_8UC3) throw std::invalid_argument("undistortImage: only CV_8UC1 and CV_8UC3 images");
        Image8u a(in.rows, in.cols, in.channels()), b;
        const size_t row = (size_t)in.cols * in.channels(), in_step = static_cast<size_t>(in.step);
        for (int r = 0; r < in.rows; ++r) std::memcpy(a.data.data() + r * row, in.data + r * in_step, row);
        Matrix3d Kp;
        for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) Kp(r, c) = K(r, c);
        undistortImage(a, b, lens, Kp);
        out.create(in.rows, in.cols, in.type());
        const size_t out_step = static_cast<size_t>(out.step);
        for (int r = 0; r < b.rows; ++r) std::memcpy(out.data + r * out_step, b.data.data() + r * row, row);
    }
    /* the cv::Mat form of the overload with a new camera matrix and size; outImg is create()d out_height x out_width (the size of
     * inImg when both are 0) */
    template <class MatT = cv::Mat>
    static void undistortImage(const cv::Mat& inImg, cv::Mat& outImg, const LensDistortion& lens, const Eigen::Matrix3d& K, const Eigen::Matrix3d& newK,
                               int out_width, int out_height)
    {
        const MatT& in = inImg;
        MatT& out = outImg;
        if (in.type() != CV_8UC1 && in.type() != CV_8UC3) throw std::invalid_argument("undistortImage: only CV_8UC1 and CV_8UC3 images");
        Image8u a(in.rows, in.cols, in.channels()), b;
        const size_t row = (size_t)in.cols * in.channels(), in_step = static_cast<size_t>(in.step);
        for (int r = 0; r < in.rows; ++r) std::memcpy(a.data.data() + r * row, in.data + r * in_step, row);
        Matrix3d Kp, nKp;
        for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) { Kp(r, c) = K(r, c); nKp(r, c) = newK(r, c); }
        undistortImage(a, b, lens, Kp, nKp, out_width, out_height);
        out.create(b.rows, b.cols, in.type());
        const size_t out_row = (size_t)b.cols * b.channels, out_step = static_cast<size_t>(out.step);
        for (int r = 0; r < b.rows; ++r) std::memcpy(out.data + r * out_step, b.data.data() + r * out_row, out_row);
    }
#endif

    /* --- additions (not in the reference) --- */
    const Line3DStats& stats() const;
    const char* lastError() const;     /* empty string if the last call succeeded */
    void setVerbose(bool v);
    /* Multi-GPU matching (SURVEY.md 8e). One Line3D per GPU / process, every one fed the same images. With world > 1
     * matchImages evaluates only this rank's contiguous, cost-balanced share of the view pairs and then calls
     * `exchange(user, counts_dev, recs_dev, row_bounds, world, knn)`: rank r owns rows [row_bounds[r], row_bounds[r+1]) of
     * counts (int32 per row) and recs (knn * 24 B per row: `knn` is the row stride of recs_dev), both DEVICE pointers; on return
     * every rank must hold all rows (an NCCL broadcast per owner; line3dpp_b200/dist.py does it with torch.distributed). Scoring,
     * affinity, diffusion and clustering then run replicated, so every rank ends with the single-GPU result bit for bit. Return 0
     * on success.
     * 1 <= kNN <= 32: one call, knn = kNN.  kNN <= 0 (keep all matches) and kNN > 32: the stride is only known once every row's
     * count is, so there are two calls.  The first has knn = 0 and moves only the counts (recs is 0 B per row).  Every rank then
     * re-lays its rows at the longest row of the whole job (after the cut to kNN when kNN > 32), and the second call has knn = that
     * stride and a recs_dev that may differ from the first call's; it must move the records (the counts may move again).  A non-zero return
     * from either call fails matchImages.
     * With several devices per Line3D, they split this rank's share and gather it on the primary before the exchange, which then
     * sees the primary's buffers. */
    typedef int (*MatchExchangeFn)(void* user, void* counts_dev, void* recs_dev, const long long* row_bounds, int world, int knn);
    void setShard(int rank, int world, MatchExchangeFn exchange, void* user);
    struct Impl;
    Impl* impl() { return p_; }        /* for the C wrapper used by the tests */
private:
    Impl* p_;
};

}  // namespace L3DPP
#endif
