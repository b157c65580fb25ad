// C wrapper over the reference's own rtabmap::GeodeticCoords (corelib/src/GeodeticCoords.cpp compiled against the stand-ins of
// oracle/refstubs/geodetic/ into _ref/libref_geodetic.so by oracle/geodetic.mk).  TEST INFRASTRUCTURE ONLY: the checker the GPS
// filter of oracle/gps_py.py and the engine's geocentric points are compared against.
#include "rtabmap/core/GeodeticCoords.h"

extern "C" {

// GeodeticCoords(latitude, longitude, altitude).toGeocentric_WGS84() -> out[3]
void ref_geo_geocentric(double latitude, double longitude, double altitude, double * out)
{
	const cv::Point3d p = rtabmap::GeodeticCoords(latitude, longitude, altitude).toGeocentric_WGS84();
	out[0] = p.x;
	out[1] = p.y;
	out[2] = p.z;
}

// GeodeticCoords::Geocentric_WGS84ToENU_WGS84(point, origin_point, GeodeticCoords(latitude, longitude, altitude)) -> out[3]
void ref_geo_enu(const double * point, const double * origin_point, double latitude, double longitude, double altitude, double * out)
{
	const cv::Point3d p = rtabmap::GeodeticCoords::Geocentric_WGS84ToENU_WGS84(cv::Point3d(point[0], point[1], point[2]),
	                                                                          cv::Point3d(origin_point[0], origin_point[1], origin_point[2]),
	                                                                          rtabmap::GeodeticCoords(latitude, longitude, altitude));
	out[0] = p.x;
	out[1] = p.y;
	out[2] = p.z;
}

} // extern "C"
