// ORB_OCTREE_B200 — rtabmap::Feature2D for Kp/DetectorStrategy=10 (ORB-OCTREE, rtabmap::ORBOctree) backed by liblcd_b200.so.
//
// Feature2D::create (corelib/src/Features2d.cpp:617) gets one more case: `case Feature2D::kFeatureOrbOctree: return gpu ?
// new ORB_OCTREE_B200(p) : new ORBOctree(p);`.  Same structure as GFTT_ORB_B200: generateKeypointsImpl runs detection and description
// in one engine call (the engine is switched to ORB-OCTREE with lcd_detector_set_orb_octree), generateDescriptorsImpl hands out the
// descriptors of that detection, as ORBOctree::generateDescriptorsImpl does (Features2d.cpp:2558-2566).  The mask goes to the engine,
// which applies it after detection at the keypoints' truncated coordinates as ORBOctree does (:2527-2549).  Parameter values the engine
// refuses (ORB/PatchSize other than 31, ORB/EdgeThreshold under 19, more than 8 levels, a scale factor <= 1) make every detection log
// the error and return no keypoints.
#include <rtabmap/core/Features2d.h>
#include <rtabmap/utilite/ULogger.h>
#include "lcd_b200.h"

namespace rtabmap {

class ORB_OCTREE_B200 : public Feature2D
{
public:
	explicit ORB_OCTREE_B200(const ParametersMap & parameters = ParametersMap()) : Feature2D(parameters), e_(0), ok_(false), min_threshold_(7), n_(0)
	{
		// Parameters.h:303, :307, :320-326
		p_.n_features = 1000; p_.n_levels = 3; p_.scale_factor = 2.0f; p_.edge_threshold = 19; p_.fast_threshold = 20; p_.patch_size = 31;
		p_.min_depth = 0; p_.max_depth = 0; p_.depth_as_mask = 1; p_.fx = p_.fy = 1; p_.cx = p_.cy = 0;
		lcd_config c;
		c.device = 0; c.desc_type = LCD_DESC_U8; c.desc_dim = 32; c.max_words = 1024; c.max_signatures = 1024; c.max_queries = 4096; c.max_batch = 1;
		e_ = lcd_create(&c);
		if (!e_) UERROR("B200 ORB-OCTREE engine: %s", lcd_last_error(0));
		parseParameters(parameters);
	}
	~ORB_OCTREE_B200() override { lcd_destroy(e_); }
	Feature2D::Type getType() const override { return kFeatureOrbOctree; }

	void parseParameters(const ParametersMap & parameters) override
	{
		Feature2D::parseParameters(parameters);
		Parameters::parse(parameters, "ORB/ScaleFactor", p_.scale_factor);     // Features2d.cpp:2500
		Parameters::parse(parameters, "ORB/NLevels", p_.n_levels);             // :2501
		Parameters::parse(parameters, "ORB/PatchSize", p_.patch_size);         // :2502
		Parameters::parse(parameters, "ORB/EdgeThreshold", p_.edge_threshold); // :2503
		Parameters::parse(parameters, "FAST/Threshold", p_.fast_threshold);    // :2505
		Parameters::parse(parameters, "FAST/MinThreshold", min_threshold_);   // :2506
		p_.n_features = getMaxFeatures();
		ok_ = e_ && lcd_detector_set_orb_octree(e_, min_threshold_) == LCD_OK;
		if (e_ && !ok_) UERROR("%s", lcd_last_error(e_));
	}

private:
	std::vector<cv::KeyPoint> generateKeypointsImpl(const cv::Mat & image, const cv::Rect & roi, const cv::Mat & mask) override
	{
		std::vector<cv::KeyPoint> out;
		n_ = 0;
		if (!ok_ || image.empty()) return out;
		if (roi.x != 0 || roi.y != 0 || roi.width != image.cols || roi.height != image.rows)
		{
			UERROR("ORB_OCTREE_B200 works on whole images (Kp/RoiRatios and Kp/GridRows/Cols must stay at their defaults)");
			return out;
		}
		const int cap = p_.n_features;
		std::vector<lcd_keypoint> kp(cap);
		desc_ = cv::Mat(cap, 32, CV_8U);
		const int rc = lcd_orb_detect_describe(e_, 1, image.data, image.cols, image.rows, image.channels(), mask.empty() ? 0 : mask.data,
		                                       mask.empty() ? LCD_DEPTH_NONE : LCD_DEPTH_MASK_U8, &p_, cap, kp.data(), desc_.data, 0, &n_);
		if (rc != LCD_OK)
		{
			UERROR("%s", lcd_last_error(e_));
			n_ = 0;
			return out;
		}
		out.resize(n_);
		for (int i = 0; i < n_; ++i)
		{
			out[i].pt.x = kp[i].x; out[i].pt.y = kp[i].y; out[i].size = kp[i].size; out[i].angle = kp[i].angle;
			out[i].response = kp[i].response; out[i].octave = kp[i].octave;
		}
		return out;
	}

	cv::Mat generateDescriptorsImpl(const cv::Mat &, std::vector<cv::KeyPoint> & keypoints) const override
	{
		if ((int)keypoints.size() != n_) UWARN("ORB_OCTREE_B200: descriptors requested for %d keypoints, the last detection found %d", (int)keypoints.size(), n_);
		return n_ ? desc_.rowRange(0, n_) : cv::Mat();
	}

	lcd_engine * e_;
	lcd_orb_params p_;
	bool ok_;
	int min_threshold_;
	cv::Mat desc_;
	int n_;
};

Feature2D * createOrbOctreeB200(const ParametersMap & parameters) { return new ORB_OCTREE_B200(parameters); }

} // namespace rtabmap
