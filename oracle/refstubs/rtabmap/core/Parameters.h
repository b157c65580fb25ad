// Stand-in for rtabmap::Parameters with only the Bayes/* keys the reference's BayesFilter.cpp reads.  TEST INFRASTRUCTURE ONLY.
//
// The keys and their defaults are not restated here: oracle/Makefile extracts the Bayes lines of the reference's own
// Parameters.h into _ref/gen/bayes_params.inc, and the two macros below turn each line into its key and default accessors.
#pragma once
#include <map>
#include <sstream>
#include <string>

namespace rtabmap {

typedef std::map<std::string, std::string> ParametersMap;

#define RTABMAP_PARAM(PREFIX, NAME, TYPE, DEFAULT_VALUE, DESCRIPTION) \
	static std::string k##PREFIX##NAME() { return std::string(#PREFIX "/" #NAME); } \
	static TYPE default##PREFIX##NAME() { return (TYPE)DEFAULT_VALUE; }
#define RTABMAP_PARAM_STR(PREFIX, NAME, DEFAULT_VALUE, DESCRIPTION) \
	static std::string k##PREFIX##NAME() { return std::string(#PREFIX "/" #NAME); } \
	static std::string default##PREFIX##NAME() { return DEFAULT_VALUE; }

class Parameters
{
public:
#include "bayes_params.inc"

	static bool parse(const ParametersMap & parameters, const std::string & key, bool & value)
	{
		const ParametersMap::const_iterator it = parameters.find(key);
		if (it == parameters.end()) return false;
		value = it->second == "true" || it->second == "1";
		return true;
	}
	static bool parse(const ParametersMap & parameters, const std::string & key, float & value)
	{
		const ParametersMap::const_iterator it = parameters.find(key);
		if (it == parameters.end()) return false;
		std::istringstream s(it->second);
		s.imbue(std::locale("C"));
		s >> value;
		return true;
	}
};

} // namespace rtabmap
