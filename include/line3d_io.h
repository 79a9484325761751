/* include/line3d_io.h — input formats of the reference's six frontends (SURVEY.md §8f-2): what main_*.cpp read from an SfM model
 * before they call Line3D::addImage, as library functions so that a frontend built on include/line3d.h needs no parsing code of its
 * own (csrc/line3d_sfm.cc, DESIGN.md §6b); and the reference's binary result file and segment cache (csrc/line3d_bin.cc).  Host
 * code; readPix4D triangulates through include/l3d_capi.h. */
#ifndef L3DPP_LINE3D_IO_H_
#define L3DPP_LINE3D_IO_H_
#include "line3d.h"

#include <list>
#include <string>
#include <vector>

namespace L3DPP {

/* one camera of an NVM model, ready for Line3D::addImage (main_vsfm.cpp:165-208, 225-236, 301-309) */
struct NVMCamera {
    std::string image;                     /* file name as written in the .nvm */
    float focal;                           /* cams_focals is a float vector in the reference (main_vsfm.cpp:166, 190) */
    float distortion;                      /* radial distortion coefficient; != 0: the frontend undistorts with (-d, 0, 0) */
    Matrix3d R;                            /* from the quaternion (qw qx qy qz) */
    Vector3d t, C;                         /* t = -R C */
    std::list<unsigned int> worldpoints;   /* ids of the 3D points this camera measures (neighbors_by_worldpoints = true) */
    float median_depth;                    /* median distance of those points to C; 0 if there are none (camera is skipped) */
};

/* Reads an NVM_V3 file like main_vsfm.cpp:143-250.  Returns false and sets *error on an unreadable, empty or malformed model; a
 * header that claims more cameras than the file holds is a truncated camera list. */
bool readNVM(const std::string& path, std::vector<NVMCamera>& cameras, std::string* error = 0);

/* one camera of a Bundler, COLMAP, mavmap, OpenMVG or Pix4D model, ready for Line3D::addImage.  Bundler has no K in the file (focal
 * only: build it with intrinsicsFromFocal once the image size is known, main_bundler.cpp:340-351); the others store K. */
struct SfMCamera {
    unsigned int id;                       /* camID handed to addImage: bundler / mavmap / Pix4D camera index, COLMAP IMAGE_ID, OpenMVG id_view */
    std::string image;                     /* image file name (bundler: from the optional list file, may be empty) */
    bool has_K; Matrix3d K;                /* all but Bundler */
    float focal;                           /* bundler only */
    double radial[3], tangential[2];       /* distortion the frontend undistorts with (bundler: k1 k2 0; others: per camera model) */
    Matrix3d R; Vector3d t, C;             /* x_cam = R X + t,  C = -R^T t */
    std::list<unsigned int> worldpoints;
    float median_depth;                    /* 0 if the camera sees no world point (it is skipped by the frontends) */
};

/* bundle.rd.out (+ optional image list, one file name per line) like main_bundler.cpp:143-262: rows 2 and 3 of R and t.y, t.z are
 * flipped (Bundler looks down -z). */
bool readBundler(const std::string& bundle_file, const std::string& image_list_file, std::vector<SfMCamera>& cameras, std::string* error = 0);

/* A COLMAP model like main_colmap.cpp:140-349: cameras.txt / images.txt / points3D.txt when all three exist, otherwise COLMAP's default
 * output cameras.bin / images.bin / points3D.bin (its documented little-endian layout; a point3D_id of 2^64 - 1 is "none", like -1 in
 * the text file).  Both give the same cameras, field for field: images in file order, those whose camera is unknown dropped,
 * worldpoints in observation order, the float median depth.
 * Models: SIMPLE_PINHOLE, PINHOLE, SIMPLE_RADIAL, RADIAL, OPENCV, FULL_OPENCV (radial / tangential as the reference sets them:
 * FULL_OPENCV's k4..k6 are not among them) and OPENCV_FISHEYE, SIMPLE_RADIAL_FISHEYE, RADIAL_FISHEYE (radial / tangential zero).
 * With lenses, (*lenses)[i] is camera i's full lens (LensDistortion, for Line3D::undistortImage), FULL_OPENCV's k4..k6 included;
 * without it a fisheye camera is rejected, since its distortion has nowhere to go.  FOV, THIN_PRISM_FISHEYE,
 * RAD_TAN_THIN_PRISM_FISHEYE and unknown models are rejected with an error naming the model and the camera.  Like the readers below,
 * a truncated or malformed binary file returns false with *error naming the file and the problem, never crashes the reader and never
 * makes it allocate more than the file's size warrants; ids that do not fit unsigned int are rejected. */
bool readColmap(const std::string& sfm_folder, std::vector<SfMCamera>& cameras, std::string* error = 0, std::vector<LensDistortion>* lenses = 0);

/* The mavmap, OpenMVG and Pix4D models.  Like the readers above: false with *error naming the file, the line or JSON path and the
 * problem on malformed input, which never crashes the reader and never makes it allocate more than the input's size warrants.
 * Every camera has has_K set. */

/* mavmap's result file like main_mavmap.cpp:153-250: leading '#' lines skipped, a line shorter than 28 characters ends the list, every
 * field carries a trailing comma, only the PINHOLE model; R = rotationFromRPY(roll, pitch, yaw) and [R|t] inverted (R^T, -R^T t),
 * C = the stored position; id = position in the file.  mavmap has no world points: worldpoints stays empty and median_depth 0 (the
 * frontend passes sequentialNeighbors lists with neighbors_by_worldpoints = false and matches with const_regularization_depth). */
bool readMavmap(const std::string& path, std::vector<SfMCamera>& cameras, std::string* error = 0);

/* up to num_neighbors / 2 earlier cameras, nearest first, then later cameras until num_neighbors (main_mavmap.cpp:312-321) */
std::list<unsigned int> sequentialNeighbors(unsigned int i, unsigned int n_cams, unsigned int num_neighbors);

/* one posed view for poseNeighbors: what addImage takes of it (K, R, t with x_cam = R X + t, the image size) and the depth at which
 * its virtual world points are placed; K's upper triangle (fx, skew, cx, fy, cy) is read, its last row is taken as (0, 0, 1) */
struct PoseView {
    unsigned int id;                       /* camID */
    int width, height;
    Matrix3d K, R;
    Vector3d t;
    double median_depth;                   /* mavmap: the constant regularisation depth the frontend matches with */
};

/* Visual neighbours for models without world points (mavmap, SLAM / VIO keyframes, pose-only surveys): what the world-point rule of
 * findVisualNeighborsFromWPs (line3D.cc:578-699) chooses when every view's world points are a gx x gy grid of its pixel centres at
 * median_depth, each seen by every view it projects into (l3d_pose_neighbors of include/l3d_capi.h, DESIGN.md §6d).  neighbors[i]
 * lists view i's neighbours' camIDs, ascending, for addImage under neighbors_by_worldpoints = false.  Runs on device cuda_device
 * through a context that lives for the call; returns false with *error naming the view (index and camID) and the problem for the
 * inputs l3d_pose_neighbors rejects, or without a usable device. */
bool poseNeighbors(const std::vector<PoseView>& views, unsigned int num_neighbors, std::vector<std::list<unsigned int> >& neighbors, std::string* error = 0,
                   int gx = 32, int gy = 24, int cuda_device = 0);

/* OpenMVG's sfm_data.json like main_openmvg.cpp:136-410: views, intrinsics (pinhole_radial_k1 / _k3, pinhole_brown_t2; other models
 * carry no distortion; an entry without polymorphic_name keeps the model of the entry before it, as the reference's loop does),
 * extrinsics (t = -R C, C as stored), structure (world point ids and float depths |C - X| per view, file order).  A view is returned,
 * in view order with id = id_view, when it has intrinsics and at least one world point.  The images are not looked for: a frontend
 * skips the views whose image it cannot load.  Numbers are read with a correctly rounded strtod. */
bool readOpenMVG(const std::string& sfm_data_json, std::vector<SfMCamera>& cameras, std::string* error = 0);

/* <params_folder>/<project_prefix>[_]calibrated_camera_parameters.txt and ..._tp_pix4d.txt like main_pix4d.cpp:163-420.  Every tie point
 * with more than two observations is triangulated on the GPU (l3d_triangulate_points) and every camera's median depth is taken over
 * its valid points (l3d_median_depths), on device cuda_device; without a usable device the reader returns false.  A camera is
 * returned, id = position in the camera file, when more than two of its points are valid; worldpoints is every observation of its
 * key image, duplicates included.  A key image missing from the camera file is camera 0, as the reference's std::map lookup makes it. */
bool readPix4D(const std::string& params_folder, const std::string& project_prefix, std::vector<SfMCamera>& cameras, std::string* error = 0,
               int cuda_device = 0);

/* The first step of the frontends' image loop, cv::imread(path, IMREAD_GRAYSCALE) (main_vsfm.cpp:267-306), for JPEG files: OpenCV 4.13's
 * grey bytes, decoded on the GPU (l3d_decode_jpeg_gray_u8 of include/l3d_capi.h; the subset and the rejections are listed there).
 * readJPEGSize reads the headers only (no GPU): the size after EXIF orientation.  readJPEGGray decodes one file into a 1-channel
 * image on device cuda_device.  readJPEGsGray decodes every readable file of the list in one batch; a file that cannot be read,
 * parsed or decoded leaves its image empty and its own message in (*errors)[i] (empty for the others), and makes the function return
 * false.  All three return false with *error set on failure; a context lives for the call, as in readPix4D. */
bool readJPEGSize(const std::string& path, int& width, int& height, std::string* error = 0);
bool readJPEGGray(const std::string& path, Image8u& image, std::string* error = 0, int cuda_device = 0);
bool readJPEGsGray(const std::vector<std::string>& paths, std::vector<Image8u>& images, std::vector<std::string>* errors = 0, int cuda_device = 0);

/* The same for PNG files (l3d_decode_png_gray_u8 of include/l3d_capi.h; the subset and the rejections are listed there): readPNGSize,
 * readPNGGray and readPNGsGray behave as the JPEG trio above.  readImageSize, readImageGray and readImagesGray take JPEG and PNG
 * files alike, chosen by each file's signature; readImagesGray decodes a mixed list with one JPEG batch and one PNG batch, and any
 * other file fails on its own with the reason. */
bool readPNGSize(const std::string& path, int& width, int& height, std::string* error = 0);
bool readPNGGray(const std::string& path, Image8u& image, std::string* error = 0, int cuda_device = 0);
bool readPNGsGray(const std::vector<std::string>& paths, std::vector<Image8u>& images, std::vector<std::string>* errors = 0, int cuda_device = 0);
bool readImageSize(const std::string& path, int& width, int& height, std::string* error = 0);
bool readImageGray(const std::string& path, Image8u& image, std::string* error = 0, int cuda_device = 0);
bool readImagesGray(const std::vector<std::string>& paths, std::vector<Image8u>& images, std::vector<std::string>* errors = 0, int cuda_device = 0);

/* K of main_vsfm.cpp:266-278: focal on the diagonal, principal point at the image centre (float arithmetic like the reference) */
Matrix3d intrinsicsFromFocal(float focal, int image_width, int image_height);

/* The reference's two binary files, Boost binary_oarchive layout without Boost (csrc/line3d_bin.cc, DESIGN.md §6a).  The readers
 * take input from outside the program: a malformed, truncated or foreign file returns false with *error set, never crashes and
 * never allocates more than the file's size warrants.  The writers return false with *error set when the file cannot be written. */

/* <name>.bin of save3DLinesAsBIN (line3D.cc:2690-2711): std::vector<FinalLine3D> with every double of P1 / P2 / dir, the float
 * length, the valid flag and every residual's (camID, segID).  Segments are restored bit for bit (no field is recomputed). */
bool read3DLinesBIN(const std::string& path, std::vector<FinalLine3D>& lines, std::string* error = 0);
bool write3DLinesBIN(const std::string& path, const std::vector<FinalLine3D>& lines, std::string* error = 0);

/* one view's segment cache (DataArray<float4>, line3D.cc:295-309, 363-366): (x1, y1, x2, y2) per segment in file order */
bool readSegmentCache(const std::string& path, std::vector<Vec4f>& segments, std::string* error = 0);
bool writeSegmentCache(const std::string& path, const std::vector<Vec4f>& segments, std::string* error = 0);

/* The size of the image detectLineSegments hands to line detection (line3D.cc:271-289): out = (w, h), or the size
 * cv::resize(img, out, Size(), s, s) gives with s = float(max_img_width) / float(max(w, h)) when max_img_width > 0 and the larger side
 * exceeds it.  Returns whether the image is resized; *scale (optional) = s, or 1.  The one place this rounding is decided: the
 * segment cache's file name and the GPU image preparation (l3d_image_prep_size) both call it. */
bool preparedImageSize(int w, int h, int max_img_width, int& out_w, int& out_h, float* scale = 0);

/* <output_folder>/L3D++_data/segments_L3D++_<camID>_<w>x<h>_3000.bin (line3D.cc:271-300).  <w>x<h> is preparedImageSize's.  The
 * suffix is L3D_DEF_MAX_NUM_SEGMENTS, whatever max_line_segments is. */
std::string segmentCachePath(const std::string& output_folder, unsigned int camID, int image_width, int image_height, int max_img_width);

}  // namespace L3DPP
#endif
