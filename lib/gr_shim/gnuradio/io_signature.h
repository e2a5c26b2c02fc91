// gr_shim: stand-in for <gnuradio/io_signature.h> (compile-only, see README.md)
#ifndef GR_SHIM_IO_SIGNATURE_H
#define GR_SHIM_IO_SIGNATURE_H
#include <boost/shared_ptr.hpp>
#include <vector>
namespace gr {
class io_signature
{
public:
    typedef boost::shared_ptr<io_signature> sptr;
    static sptr make(int min_streams, int max_streams, int sizeof_stream_item)
    {
        return sptr(new io_signature(min_streams, max_streams, std::vector<int>(1, sizeof_stream_item)));
    }
    static sptr make2(int min_streams, int max_streams, int s1, int s2)
    {
        std::vector<int> v;
        v.push_back(s1); v.push_back(s2);
        return sptr(new io_signature(min_streams, max_streams, v));
    }
    static sptr make3(int min_streams, int max_streams, int s1, int s2, int s3)
    {
        std::vector<int> v;
        v.push_back(s1); v.push_back(s2); v.push_back(s3);
        return sptr(new io_signature(min_streams, max_streams, v));
    }
    static sptr makev(int min_streams, int max_streams, const std::vector<int> &sizeof_stream_items)
    {
        return sptr(new io_signature(min_streams, max_streams, sizeof_stream_items));
    }
    int min_streams() const { return d_min; }
    int max_streams() const { return d_max; }
    int sizeof_stream_item(int index) const
    {
        return d_sizes[index < (int)d_sizes.size() ? index : (int)d_sizes.size() - 1];
    }

private:
    io_signature(int mn, int mx, const std::vector<int> &s) : d_min(mn), d_max(mx), d_sizes(s) {}
    int d_min, d_max;
    std::vector<int> d_sizes;
};
}  // namespace gr
#endif
